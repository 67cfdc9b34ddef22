"""oracle_euclid/euclid.py -- TEST INFRASTRUCTURE ONLY (ctypes doors to the two CPU checkers of
manhattan_spatial_dist = False, the Euclidean spatial term).

* ``Port`` : oracle_euclid/liboracle_euclid.so -- the plain-C restatement (euclid_oracle.c on top of oracle/slic_oracle.c)
* ``Ref``  : oracle_euclid/_ref/libfslic_ref_euclid.so -- the unmodified reference behind euclid_ref_shim.cpp; exists
             wherever it was built (FSLIC_REFERENCE naming a fast-slic checkout at build time).

Same call signatures as oracle.oracle.Port / Ref, without the flag: every call here is the Euclidean one.  Only tests/,
tests/golden/make_euclid_golden.py and tools/spatial_dist_probe.py import this module; the product never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.oracle import CLUSTER_DTYPE, Port as _ManhattanPort

_HERE = os.path.dirname(os.path.abspath(__file__))
_u8p = C.POINTER(C.c_uint8)
_u16p = C.POINTER(C.c_uint16)


def _p(arr, typ):
    return None if arr is None else arr.ctypes.data_as(typ)


def build(force=False):
    """Compile liboracle_euclid.so (always possible) and _ref (only where FSLIC_REFERENCE names a fast-slic checkout)."""
    if force or not os.path.exists(os.path.join(_HERE, "liboracle_euclid.so")):
        subprocess.check_call(["make", "-C", _HERE, "liboracle_euclid.so"], stdout=subprocess.DEVNULL)
    ref = os.environ.get("FSLIC_REFERENCE")
    if ref and (force or not os.path.exists(os.path.join(_HERE, "_ref", "libfslic_ref_euclid.so"))):
        subprocess.check_call(["make", "-C", _HERE, "ref", "REF=" + ref], stdout=subprocess.DEVNULL)


class Port:
    """Plain-C restatement with the Euclidean spatial term."""

    def __init__(self):
        build()
        self.lib = C.CDLL(os.path.join(_HERE, "liboracle_euclid.so"))
        self.lib.orce_hypotf_mismatches.restype = C.c_long
        self._plain = _ManhattanPort()

    def initialize(self, image, K):
        return self._plain.initialize(image, K)  # the seeding does not depend on the flag

    def hypotf_mismatches(self, lo, hi):
        """Offsets lo <= a, b <= hi on which libm's hypotf differs from the CUDA kernels' euclid_dist."""
        return int(self.lib.orce_hypotf_mismatches(int(lo), int(hi)))

    def iterate(self, image, clusters, max_iter=10, compactness=10.0, min_size_factor=0.25, stride=3,
                convert_to_lab=True, stages=False, preemptive=False, preemptive_thres=0.05):
        image = np.ascontiguousarray(image)
        H, W, _ = image.shape
        out = np.zeros((H, W), np.uint16)
        quad = np.zeros((H, W, 4), np.uint8) if stages else None
        pre = np.zeros((H, W), np.uint16) if stages else None
        self.lib.orce_iterate_preemptive(H, W, len(clusters), _p(image, _u8p), clusters.ctypes.data_as(C.c_void_p),
                                         _p(out, _u16p), max_iter, C.c_float(compactness), C.c_float(min_size_factor),
                                         stride, int(convert_to_lab), int(bool(preemptive)), C.c_float(preemptive_thres),
                                         _p(quad, _u8p), _p(pre, _u16p))
        return (out, quad, pre) if stages else out

    def iterate_real(self, variant, image, clusters, max_iter=10, compactness=10.0, min_size_factor=0.25, stride=3,
                     convert_to_lab=True, stages=False):
        image = np.ascontiguousarray(image)
        H, W, _ = image.shape
        out = np.zeros((H, W), np.uint16)
        pre = np.zeros((H, W), np.uint16)
        self.lib.orce_iterate_real(int(variant), H, W, len(clusters), _p(image, _u8p), clusters.ctypes.data_as(C.c_void_p),
                                   _p(out, _u16p), max_iter, C.c_float(compactness), C.c_float(min_size_factor), stride,
                                   int(convert_to_lab), _p(pre, _u16p))
        return (out, pre) if stages else out


class Ref:
    """The unmodified reference with manhattan_spatial_dist = False (standard or x64/avx2 arch)."""

    @staticmethod
    def available():
        return os.path.exists(os.path.join(_HERE, "_ref", "libfslic_ref_euclid.so")) or \
            bool(os.environ.get("FSLIC_REFERENCE"))

    def __init__(self):
        build()
        self.lib = C.CDLL(os.path.join(_HERE, "_ref", "libfslic_ref_euclid.so"))
        assert self.lib.refe_sizeof_cluster() == CLUSTER_DTYPE.itemsize

    def initialize(self, image, K):
        H, W, _ = image.shape
        clusters = np.zeros(K, CLUSTER_DTYPE)
        self.lib.refe_initialize(H, W, K, _p(np.ascontiguousarray(image), _u8p), clusters.ctypes.data_as(C.c_void_p))
        return clusters

    def iterate(self, image, clusters, max_iter=10, compactness=10.0, min_size_factor=0.25, stride=3,
                convert_to_lab=True, stages=False, arch="x64/avx2", num_threads=-1, preemptive=False,
                preemptive_thres=0.05):
        image = np.ascontiguousarray(image)
        H, W, _ = image.shape
        out = np.zeros((H, W), np.uint16)
        quad = np.zeros((H, W, 4), np.uint8) if stages else None
        pre = np.zeros((H, W), np.uint16) if stages else None
        self.lib.refe_iterate(1 if arch == "x64/avx2" else 0, H, W, len(clusters), _p(image, _u8p),
                              clusters.ctypes.data_as(C.c_void_p), _p(out, _u16p), max_iter, C.c_float(compactness),
                              C.c_float(min_size_factor), stride, int(convert_to_lab), int(bool(preemptive)),
                              C.c_float(preemptive_thres), num_threads, _p(quad, _u8p), _p(pre, _u16p))
        return (out, quad, pre) if stages else out

    def iterate_real(self, variant, image, clusters, max_iter=10, compactness=10.0, min_size_factor=0.25, stride=3,
                     convert_to_lab=True, stages=False, num_threads=2):
        image = np.ascontiguousarray(image)
        H, W, _ = image.shape
        out = np.zeros((H, W), np.uint16)
        pre = np.zeros((H, W), np.uint16)
        self.lib.refe_iterate_real(int(variant), H, W, len(clusters), _p(image, _u8p), clusters.ctypes.data_as(C.c_void_p),
                                   _p(out, _u16p), max_iter, C.c_float(compactness), C.c_float(min_size_factor), stride,
                                   int(convert_to_lab), num_threads, _p(pre, _u16p))
        return (out, pre) if stages else out
