"""oracle/recorder.py -- TEST INFRASTRUCTURE ONLY: the reference's debug_mode report.

``RecorderRef`` opens oracle/_ref/libfslic_ref_recorder.so (oracle/recorder.mk + oracle/recorder_shim.cpp), the
unmodified reference driven with debug_mode = true; it exists wherever it was built.  The product never imports this.
"""
import ctypes as C
import os

import numpy as np

from .oracle import CLUSTER_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_ref", "libfslic_ref_recorder.so")

# recorder_shim.cpp's `kind`
KINDS = {"standard": 0, "x64/avx2": 1, "real_standard": 2, "real_l2": 3, "real_noq": 4, "lsc": 5}


class RecorderRef:
    @staticmethod
    def available():
        return os.path.exists(LIB)

    def __init__(self):
        self.lib = C.CDLL(LIB)
        self.lib.refr_iterate.restype = C.c_void_p
        self.lib.refr_iterate.argtypes = [C.c_int] * 4 + [C.c_void_p] * 3 + [C.c_int, C.c_float, C.c_float, C.c_int,
                                                                            C.c_int, C.c_int, C.c_int, C.c_float,
                                                                            C.c_int, C.POINTER(C.c_size_t)]
        self.lib.refr_free.argtypes = [C.c_void_p]

    def iterate(self, kind, image, clusters, max_iter=10, compactness=10.0, min_size_factor=0.25, stride=3,
                convert_to_lab=True, manhattan=True, preemptive=False, preemptive_thres=0.05, num_threads=1):
        """-> (report bytes, labels u16[H, W]); `clusters` (CLUSTER_DTYPE[K]) is updated in place."""
        image = np.ascontiguousarray(image)
        assert clusters.dtype == CLUSTER_DTYPE and clusters.flags["C_CONTIGUOUS"]
        H, W, _ = image.shape
        out = np.zeros((H, W), np.uint16)
        n = C.c_size_t()
        p = self.lib.refr_iterate(KINDS[kind], H, W, len(clusters), image.ctypes.data, clusters.ctypes.data,
                                  out.ctypes.data, int(max_iter), float(compactness), float(min_size_factor),
                                  int(stride), int(bool(convert_to_lab)), int(bool(manhattan)), int(bool(preemptive)),
                                  float(preemptive_thres), int(num_threads), C.byref(n))
        try:
            rep = C.string_at(p, n.value)
        finally:
            self.lib.refr_free(p)
        return rep, out
