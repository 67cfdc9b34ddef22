"""oracle_lsc/lsc.py -- TEST INFRASTRUCTURE ONLY (ctypes doors to the two CPU checkers of LSC, linear spectral
clustering).

* ``Port`` : oracle_lsc/liboracle_lsc.so -- the plain-C restatement (lsc_oracle.c on top of oracle/slic_oracle.c);
             single-threaded, like the only reference run whose result is defined
* ``Ref``  : oracle_lsc/_ref/libfslic_ref_lsc.so -- the unmodified reference's ContextLSC behind lsc_ref_shim.cpp;
             exists wherever it was built (FSLIC_REFERENCE naming a fast-slic checkout at build time)

``iterate_lsc`` returns the final labels; with ``stages=True`` also a dict of the stage buffers: ``pre`` (pre-CCA
labels u16[H, W]), ``means`` (float32[10]), ``weights`` (float32[H, W]), ``cinit`` / ``cfinal`` (centroid features
float32[K, 10] after before_iteration / at the end).  Only tests/, tests/golden/make_lsc_golden.py and
tools/lsc_probe.py import this module; the product never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.oracle import CLUSTER_DTYPE, Port as _ManhattanPort

_HERE = os.path.dirname(os.path.abspath(__file__))
_u8p = C.POINTER(C.c_uint8)
_u16p = C.POINTER(C.c_uint16)
_f32p = C.POINTER(C.c_float)


def _p(arr, typ):
    return None if arr is None else arr.ctypes.data_as(typ)


def build(force=False):
    """Compile liboracle_lsc.so (always possible) and _ref (only where FSLIC_REFERENCE names a fast-slic checkout)."""
    if force or not os.path.exists(os.path.join(_HERE, "liboracle_lsc.so")):
        subprocess.check_call(["make", "-C", _HERE, "liboracle_lsc.so"], stdout=subprocess.DEVNULL)
    ref = os.environ.get("FSLIC_REFERENCE")
    if ref and (force or not os.path.exists(os.path.join(_HERE, "_ref", "libfslic_ref_lsc.so"))):
        subprocess.check_call(["make", "-C", _HERE, "ref", "REF=" + ref], stdout=subprocess.DEVNULL)


def _buffers(H, W, K, stages):
    out = np.zeros((H, W), np.uint16)
    if not stages:
        return out, None
    return out, dict(pre=np.zeros((H, W), np.uint16), means=np.zeros(10, np.float32),
                     weights=np.zeros((H, W), np.float32), cinit=np.zeros((K, 10), np.float32),
                     cfinal=np.zeros((K, 10), np.float32))


def _stage_ptrs(st):
    if st is None:
        return (None,) * 5
    return (_p(st["pre"], _u16p), _p(st["means"], _f32p), _p(st["weights"], _f32p), _p(st["cinit"], _f32p),
            _p(st["cfinal"], _f32p))


class Port:
    """Plain-C restatement of ContextLSC with one thread."""

    def __init__(self):
        build()
        self.lib = C.CDLL(os.path.join(_HERE, "liboracle_lsc.so"))
        self._plain = _ManhattanPort()

    def initialize(self, image, K):
        return self._plain.initialize(image, K)  # BaseContext::initialize_clusters, shared by every context

    def iterate_lsc(self, image, clusters, max_iter=10, compactness=10.0, min_size_factor=0.25, stride=3,
                    convert_to_lab=True, stages=False):
        image = np.ascontiguousarray(image)
        H, W, _ = image.shape
        out, st = _buffers(H, W, len(clusters), stages)
        self.lib.orcl_iterate_lsc(H, W, len(clusters), _p(image, _u8p), clusters.ctypes.data_as(C.c_void_p),
                                  _p(out, _u16p), max_iter, C.c_float(compactness), C.c_float(min_size_factor), stride,
                                  int(convert_to_lab), *_stage_ptrs(st))
        return (out, st) if stages else out


class Ref:
    """The unmodified reference's ContextLSC (arch "standard"); `num_threads` is the context's field (1 by default: the
    only count whose result does not depend on the machine and the scheduler)."""

    @staticmethod
    def available():
        return os.path.exists(os.path.join(_HERE, "_ref", "libfslic_ref_lsc.so")) or \
            bool(os.environ.get("FSLIC_REFERENCE"))

    def __init__(self):
        build()
        self.lib = C.CDLL(os.path.join(_HERE, "_ref", "libfslic_ref_lsc.so"))
        assert self.lib.refl_sizeof_cluster() == CLUSTER_DTYPE.itemsize
        self._plain = _ManhattanPort()

    def initialize(self, image, K):
        return self._plain.initialize(image, K)

    def iterate_lsc(self, image, clusters, max_iter=10, compactness=10.0, min_size_factor=0.25, stride=3,
                    convert_to_lab=True, stages=False, num_threads=1, manhattan_spatial_dist=True):
        image = np.ascontiguousarray(image)
        H, W, _ = image.shape
        out, st = _buffers(H, W, len(clusters), stages)
        self.lib.refl_iterate_lsc(H, W, len(clusters), _p(image, _u8p), clusters.ctypes.data_as(C.c_void_p),
                                  _p(out, _u16p), max_iter, C.c_float(compactness), C.c_float(min_size_factor), stride,
                                  int(convert_to_lab), int(bool(manhattan_spatial_dist)), int(num_threads),
                                  *_stage_ptrs(st))
        return (out, st) if stages else out
