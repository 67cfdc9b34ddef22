"""oracle_crf/crf.py -- TEST INFRASTRUCTURE ONLY (ctypes doors to the two CPU checkers of the SimpleCRF).

* ``Port`` : oracle_crf/liboracle_crf.so -- the plain-C restatement (crf_oracle.c); the frames are kept here in Python
* ``Ref``  : oracle_crf/_ref/libfslic_ref_crf.so -- the unmodified reference's SimpleCRF behind crf_ref_shim.cpp;
             exists wherever it was built (FSLIC_REFERENCE naming a fast-slic checkout at build time)

Both have the same surface: push / pop / first / last, per-frame setters and getters by time, initialize, inference
and the two pairwise energies.  Arrays are numpy: clusters oracle.oracle.CLUSTER_DTYPE[N], adjacency as CSR (offsets
int32[rows + 1], neighbours int32), unaries / q float32[C, N].  Only tests/, tests/golden/make_crf_golden.py and
tools/crf_probe.py import this module; the product never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.oracle import CLUSTER_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
PARAM_NAMES = ("spatial_w", "temporal_w", "spatial_srgb", "temporal_srgb", "spatial_sxy", "spatial_smooth_w",
               "spatial_smooth_sxy")
DEFAULT_PARAMS = dict(zip(PARAM_NAMES, (10.0, 10.0, 13.0, 13.0, 80.0, 0.0, 3.0)))


class Params(C.Structure):
    _fields_ = [(n, C.c_float) for n in PARAM_NAMES]


def build(force=False):
    if force or not os.path.exists(os.path.join(_HERE, "liboracle_crf.so")):
        subprocess.check_call(["make", "-C", _HERE, "liboracle_crf.so"], stdout=subprocess.DEVNULL)
    ref = os.environ.get("FSLIC_REFERENCE")
    if ref and (force or not os.path.exists(os.path.join(_HERE, "_ref", "libfslic_ref_crf.so"))):
        subprocess.check_call(["make", "-C", _HERE, "ref", "REF=" + ref], stdout=subprocess.DEVNULL)


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def blank_clusters(N):
    cl = np.zeros(N, CLUSTER_DTYPE)
    cl["num_members"] = 1
    return cl


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(os.path.join(_HERE, "liboracle_crf.so"))
        L.orcl_crf_spatial_energy.restype = C.c_float
        L.orcl_crf_temporal_energy.restype = C.c_float
        L.orcl_crf_spatial_energy.argtypes = L.orcl_crf_temporal_energy.argtypes = [C.c_void_p, C.c_void_p,
                                                                                     C.POINTER(Params)]
        L.orcl_crf_mask.argtypes = [C.c_size_t, C.c_size_t, C.c_void_p, C.c_float, C.c_void_p]
        L.orcl_crf_unbiased.argtypes = [C.c_size_t, C.c_size_t, C.c_void_p]
        L.orcl_crf_proba.argtypes = L.orcl_crf_reset.argtypes = [C.c_size_t, C.c_void_p, C.c_void_p]
        L.orcl_crf_inference.argtypes = [C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.POINTER(Params), C.c_longlong, C.c_void_p]
        L.orcl_expf_range.argtypes = [C.c_uint32, C.c_longlong, C.c_void_p]
        L.orcl_logf_range.argtypes = [C.c_uint32, C.c_longlong, C.c_void_p]
        _lib = L
    return _lib


def glibc_expf_range(first, n):
    """glibc's expf over the float bit patterns first .. first + n - 1."""
    out = np.empty(n, np.float32)
    lib().orcl_expf_range(first, n, _vp(out))
    return out


def glibc_logf_range(first, n):
    """glibc's logf over the float bit patterns first .. first + n - 1."""
    out = np.empty(n, np.float32)
    lib().orcl_logf_range(first, n, _vp(out))
    return out


class _Frame:
    def __init__(self, time, C_, N):
        self.time = time
        self.clusters = blank_clusters(N)
        self.off = np.zeros(N + 1, np.int32)
        self.nbr = np.zeros(0, np.int32)
        self.unary = np.zeros((C_, N), np.float32)
        self.q = np.zeros((C_, N), np.float32)


class Port:
    """Plain-C restatement; frames in a Python list in time order."""

    def __init__(self, num_classes, num_nodes):
        self.L = lib()
        self.C, self.N = num_classes, num_nodes
        self.params = dict(DEFAULT_PARAMS)
        self.frames = []
        self.next_time = 0

    def _p(self):
        return Params(*[self.params[n] for n in PARAM_NAMES])

    def _f(self, t):
        for f in self.frames:
            if f.time == t:
                return f
        raise IndexError("Time out of range")

    def set_params(self, **kw):
        for k, v in kw.items():
            self.params[k] = float(np.float32(v))

    def push(self):
        self.frames.append(_Frame(self.next_time, self.C, self.N))
        self.next_time += 1
        return self.next_time - 1

    def pop(self):
        return self.frames.pop(0).time if self.frames else -1

    def first(self):
        return self.frames[0].time if self.frames else -1

    def last(self):
        return self.frames[-1].time if self.frames else -1

    def set_clusters(self, t, cl):
        self._f(t).clusters = np.array(cl, CLUSTER_DTYPE)

    def set_connectivity(self, t, off, nbr):
        f = self._f(t)
        rows = len(off) - 1
        lists = [nbr[off[i]:off[i + 1]] for i in range(rows)] + [f.nbr[f.off[i]:f.off[i + 1]]
                                                                  for i in range(rows, self.N)]
        f.off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
        f.nbr = np.concatenate([np.zeros(0, np.int32)] + [np.asarray(x, np.int32) for x in lists])

    def set_unary(self, t, u):
        self._f(t).unary = _f32(u).copy()

    def get_unary(self, t):
        return self._f(t).unary.copy()

    def set_unbiased(self, t):
        f = self._f(t)
        self.L.orcl_crf_unbiased(self.C, self.N, _vp(f.unary))

    def set_mask(self, t, classes, confidence):
        f = self._f(t)
        cls = np.ascontiguousarray(classes, np.int32)
        self.L.orcl_crf_mask(self.C, self.N, _vp(cls), C.c_float(confidence), _vp(f.unary))

    def set_proba(self, t, p):
        f = self._f(t)
        p = _f32(p)
        self.L.orcl_crf_proba(self.C * self.N, _vp(p), _vp(f.unary))

    def get_inferred(self, t):
        return self._f(t).q.copy()

    def reset_inferred(self, t):
        f = self._f(t)
        self.L.orcl_crf_reset(self.C * self.N, _vp(f.unary), _vp(f.q))

    def initialize(self):
        for f in self.frames:
            self.reset_inferred(f.time)

    def inference(self, max_iter):
        if max_iter == 0:
            return
        if not self.frames:
            raise IndexError("Time out of range")
        T = len(self.frames)
        ptrs = lambda xs: (C.c_void_p * T)(*[_vp(x) for x in xs])  # noqa: E731
        fr = self.frames
        work = np.zeros(2 * T * self.C * self.N + self.N + 1, np.float32)
        self.L.orcl_crf_inference(T, self.C, self.N, ptrs([f.clusters for f in fr]), ptrs([f.off for f in fr]),
                                  ptrs([f.nbr if len(f.nbr) else np.zeros(1, np.int32) for f in fr]),
                                  ptrs([f.unary for f in fr]), ptrs([f.q for f in fr]), C.byref(self._p()),
                                  max_iter, _vp(work))

    def spatial(self, t, i, j):
        if i == j:
            return np.float32(0)
        cl = self._f(t).clusters
        return np.float32(self.L.orcl_crf_spatial_energy(_vp(cl[i:i + 1]), _vp(cl[j:j + 1]), C.byref(self._p())))

    def temporal(self, t, i, other):
        if t == other:
            return np.float32(0)
        a, b = self._f(t).clusters, self._f(other).clusters
        return np.float32(self.L.orcl_crf_temporal_energy(_vp(a[i:i + 1]), _vp(b[i:i + 1]), C.byref(self._p())))


class Ref:
    """The unmodified reference's SimpleCRF (src/simple-crf.cpp) through crf_ref_shim.cpp."""

    @staticmethod
    def available():
        return os.path.exists(os.path.join(_HERE, "_ref", "libfslic_ref_crf.so")) or \
            bool(os.environ.get("FSLIC_REFERENCE"))

    def __init__(self, num_classes, num_nodes):
        build()
        L = C.CDLL(os.path.join(_HERE, "_ref", "libfslic_ref_crf.so"))
        assert L.refc_sizeof_cluster() == CLUSTER_DTYPE.itemsize
        L.refc_new.restype = C.c_void_p
        L.refc_new.argtypes = [C.c_size_t, C.c_size_t]
        vp, i32 = C.c_void_p, C.c_int
        for name, args in (("free", []), ("push", []), ("pop", []), ("first", []), ("last", []), ("initialize", []),
                           ("set_params", [vp]), ("set_clusters", [i32, vp]), ("set_connectivity", [i32, i32, vp, vp]),
                           ("set_unary", [i32, vp]), ("get_unary", [i32, vp]), ("set_unbiased", [i32]),
                           ("set_mask", [i32, vp, C.c_float]), ("set_proba", [i32, vp]), ("get_inferred", [i32, vp]),
                           ("reset_inferred", [i32]), ("inference", [C.c_longlong]), ("spatial", [i32, i32, i32]),
                           ("temporal", [i32, i32, i32])):
            getattr(L, "refc_" + name).argtypes = [vp] + args
        L.refc_spatial.restype = L.refc_temporal.restype = C.c_float
        self.L = L
        self.C, self.N = num_classes, num_nodes
        self.h = C.c_void_p(L.refc_new(num_classes, num_nodes))
        self.params = dict(DEFAULT_PARAMS)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.refc_free(self.h)
            self.h = None

    def set_params(self, **kw):
        for k, v in kw.items():
            self.params[k] = float(np.float32(v))
        self.L.refc_set_params(self.h, C.byref(Params(*[self.params[n] for n in PARAM_NAMES])))

    def _check(self, t):
        if not (self.first() <= t <= self.last()) or self.first() < 0:
            raise IndexError("Time out of range")

    def push(self):
        return self.L.refc_push(self.h)

    def pop(self):
        return self.L.refc_pop(self.h)

    def first(self):
        return self.L.refc_first(self.h)

    def last(self):
        return self.L.refc_last(self.h)

    def set_clusters(self, t, cl):
        self._check(t)
        cl = np.ascontiguousarray(cl, CLUSTER_DTYPE)
        self.L.refc_set_clusters(self.h, t, _vp(cl))

    def set_connectivity(self, t, off, nbr):
        self._check(t)
        off = np.ascontiguousarray(off, np.int32)
        nbr = np.ascontiguousarray(nbr, np.int32).view(np.uint32) if len(nbr) else np.zeros(1, np.uint32)
        self.L.refc_set_connectivity(self.h, t, len(off) - 1, _vp(off), _vp(nbr))

    def set_unary(self, t, u):
        self._check(t)
        u = _f32(u)
        self.L.refc_set_unary(self.h, t, _vp(u))

    def get_unary(self, t):
        self._check(t)
        out = np.zeros((self.C, self.N), np.float32)
        self.L.refc_get_unary(self.h, t, _vp(out))
        return out

    def set_unbiased(self, t):
        self._check(t)
        self.L.refc_set_unbiased(self.h, t)

    def set_mask(self, t, classes, confidence):
        self._check(t)
        cls = np.ascontiguousarray(classes, np.int32)
        self.L.refc_set_mask(self.h, t, _vp(cls), C.c_float(confidence))

    def set_proba(self, t, p):
        self._check(t)
        p = _f32(p)
        self.L.refc_set_proba(self.h, t, _vp(p))

    def get_inferred(self, t):
        self._check(t)
        out = np.zeros((self.C, self.N), np.float32)
        self.L.refc_get_inferred(self.h, t, _vp(out))
        return out

    def reset_inferred(self, t):
        self._check(t)
        self.L.refc_reset_inferred(self.h, t)

    def initialize(self):
        self.L.refc_initialize(self.h)

    def inference(self, max_iter):
        if max_iter and self.first() < 0:
            raise IndexError("Time out of range")  # the reference's infer_once looks up time -1 and throws
        self.L.refc_inference(self.h, max_iter)

    def spatial(self, t, i, j):
        self._check(t)
        return np.float32(self.L.refc_spatial(self.h, t, i, j))

    def temporal(self, t, i, other):
        self._check(t)
        self._check(other)
        return np.float32(self.L.refc_temporal(self.h, t, i, other))
