"""== fast_slic.crf (csimple_crf.pyx): SimpleCRF and SimpleCRFFrame, a temporal mean-field CRF over superpixels whose
inference runs on the GPU (fast_slic_b200/csrc/crf.cuh), bit-identical to the reference's SimpleCRF.

Typical use is temporal smoothing of per-superpixel class probabilities across video frames::

    crf = SimpleCRF(num_classes, num_nodes=K)
    frame = crf.push_slic_frame(slic)       # after slic.iterate(image)
    frame.set_proba(proba)                  # float32 [C, K]
    crf.initialize(); crf.inference(5)
    q = frame.get_inferred()

Unary setters take host arrays, like the reference's memoryviews; `inference` runs asynchronously on the device and
the getters wait for it.

The CRF can also be fed from the device, with no host round trip: `SimpleCRF.push_label_frames` takes the int16 cuda
labels and uint8 [K,32] cluster records that `iterate_batch(..., return_clusters=True)` returns, and `set_proba`,
`set_mask`, the `unaries` setter and `get_inferred(out=...)` take cuda tensors::

    labels, clusters = slic.iterate_batch(images, return_clusters=True)    # cuda tensors [B,H,W], [B,K,32]
    frames = crf.push_label_frames(labels, clusters)                       # B frames
    frames[-1].set_proba(proba)                                            # float32 cuda [C, K]
    crf.initialize(); crf.inference(5)
    frames[-1].get_inferred(out=q)                                         # float32 cuda [C, K]

That work is enqueued on the CRF device's current torch stream, and every frame equals what the host path stores for
the same values, bit for bit.

`SimpleCRFGroup` drives the CRFs of many video streams together, one SimpleCRF per stream with the same num_classes,
num_nodes and device, in the same kernel launches: image b of each batch is the next frame of member b::

    crfs = [SimpleCRF(C, K) for _ in range(B)]
    group = SimpleCRFGroup(crfs)
    labels, clusters = slic.iterate_batch(images, return_clusters=True)   # [B,H,W], [B,K,32]
    group.push_label_frames(labels, clusters)                             # one frame per member
    group.set_proba(proba); group.reset_inferred()                        # float32 cuda [B, C, K]
    group.inference(5)
    group.get_inferred(out=q)                                             # float32 cuda [B, C, K]
    group.pop_frame()

Every member computes exactly what its own calls compute, and keeps its whole surface (frames, host getters,
energies, its own inference).

Where the reference reads out of bounds or crashes, this module raises instead: neighbour
indices or mask classes outside the frame raise ValueError and change nothing, and a frame handle whose frame was
popped raises IndexError.
"""
import contextlib
import ctypes as C
import operator
import threading

import numpy as np
import torch

from . import _lib
from .engine import CLUSTER_DTYPE

__all__ = ["SimpleCRF", "SimpleCRFFrame", "SimpleCRFGroup"]

_PARAM_NAMES = ("spatial_w", "temporal_w", "spatial_srgb", "temporal_srgb", "spatial_sxy", "spatial_smooth_w",
                "spatial_smooth_sxy")
_ENOFRAME = -5


class _Params(C.Structure):
    _fields_ = [(n, C.c_float) for n in _PARAM_NAMES]


_bound = False


def _L():
    global _bound
    L = _lib.lib()
    if not _bound:
        vp, i32, ll = C.c_void_p, C.c_int, C.c_longlong
        ip = C.POINTER(C.c_int)
        L.fslic_b200_crf_create.argtypes = [i32, i32, i32, C.POINTER(vp)]
        L.fslic_b200_crf_destroy.argtypes = [vp]
        L.fslic_b200_crf_get_params.argtypes = [vp, C.POINTER(_Params)]
        L.fslic_b200_crf_set_params.argtypes = [vp, C.POINTER(_Params)]
        L.fslic_b200_crf_times.argtypes = [vp, ip, ip, ip]
        L.fslic_b200_crf_push_frame.argtypes = [vp, ip]
        L.fslic_b200_crf_pop_frame.argtypes = [vp, ip]
        for name in ("set_clusters", "get_clusters", "set_unary", "get_unary", "set_proba", "get_inferred"):
            getattr(L, "fslic_b200_crf_" + name).argtypes = [vp, i32, vp]
        L.fslic_b200_crf_set_connectivity.argtypes = [vp, i32, i32, vp, vp]
        L.fslic_b200_crf_get_connectivity.argtypes = [vp, i32, vp, vp, ll]
        L.fslic_b200_crf_set_unbiased.argtypes = [vp, i32]
        L.fslic_b200_crf_set_mask.argtypes = [vp, i32, vp, C.c_float]
        L.fslic_b200_crf_reset_inferred.argtypes = [vp, i32]
        L.fslic_b200_crf_initialize.argtypes = [vp]
        L.fslic_b200_crf_inference.argtypes = [vp, C.c_ulonglong, vp]
        L.fslic_b200_crf_spatial_pairwise_energy.argtypes = [vp, i32, i32, i32, C.POINTER(C.c_float)]
        L.fslic_b200_crf_temporal_pairwise_energy.argtypes = [vp, i32, i32, vp, i32, C.POINTER(C.c_float)]
        L.fslic_b200_debug_expf_host.argtypes = [C.c_uint32, ll, vp]
        L.fslic_b200_debug_expf_device.argtypes = [i32, C.c_uint32, ll, vp, vp]
        L.fslic_b200_debug_logf_host.argtypes = [C.c_uint32, ll, vp]
        L.fslic_b200_debug_logf_device.argtypes = [i32, C.c_uint32, ll, vp, vp]
        L.fslic_b200_crfdev_push_scratch_bytes.argtypes = [i32, i32]
        L.fslic_b200_crfdev_push_scratch_bytes.restype = C.c_size_t
        L.fslic_b200_crfdev_push_label_frames.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp, C.c_size_t, vp, ip]
        for name in ("set_unary", "set_proba", "get_inferred"):
            getattr(L, "fslic_b200_crfdev_" + name).argtypes = [vp, i32, vp, vp]
        L.fslic_b200_crfdev_set_mask.argtypes = [vp, i32, vp, C.c_float, vp]
        L.fslic_b200_crfgroup_inference.argtypes = [vp, i32, C.c_ulonglong, vp]
        L.fslic_b200_crfdev_group_push_label_frames.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp, C.c_size_t, vp, ip]
        for name in ("set_proba", "get_inferred"):
            getattr(L, "fslic_b200_crfdev_group_" + name).argtypes = [vp, i32, vp, vp]
        L.fslic_b200_crfdev_group_reset_inferred.argtypes = [vp, i32, vp]
        L.fslic_b200_crfgroup_pop_frame.argtypes = [vp, i32, ip]
        _bound = True
    return L


def _check(rc):
    if rc == _ENOFRAME:
        raise IndexError(_lib.lib().fslic_b200_last_error().decode("utf-8", "replace"))
    _lib.check(rc)


_INT_MAX = 2 ** 31 - 1


def _size_t(v):
    """Cython's size_t argument conversion."""
    v = operator.index(v)
    if v < 0:
        raise OverflowError("can't convert negative value to size_t")
    if v > 2 ** 64 - 1:
        raise OverflowError("value too large to convert to size_t")
    return v


def _c_int(v):
    """Cython's int argument conversion."""
    v = operator.index(v)
    if not -_INT_MAX - 1 <= v <= _INT_MAX:
        raise OverflowError("value too large to convert to int")
    return v


def _buffer(arr, dtype, ndim, cname):
    """What a Cython typed memoryview `cname[:, ::1]` / `cname[::1]` accepts: a C-contiguous buffer of that exact item
    type and rank.  Returns the array as numpy."""
    try:
        a = np.asarray(memoryview(arr))
    except TypeError:
        raise TypeError("a bytes-like object is required, not '%s'" % type(arr).__name__)
    if a.ndim != ndim:
        raise ValueError("Buffer has wrong number of dimensions (expected %d, got %d)" % (ndim, a.ndim))
    if a.dtype != np.dtype(dtype):
        raise ValueError("Buffer dtype mismatch, expected '%s' but got '%s'" % (cname, a.dtype.name))
    if not a.flags["C_CONTIGUOUS"]:
        raise ValueError("ndarray is not C-contiguous")
    return a


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _is_cuda(x):
    """A cuda tensor takes the device path; anything else the host path, unchanged."""
    return isinstance(x, torch.Tensor) and x.is_cuda


def _device_tensor(x, device, dtype, ndim, cname):
    """A cuda tensor argument of the device path: `dtype`, rank `ndim`, on cuda:`device`; ValueError otherwise, like
    `_buffer`'s errors."""
    if x.dtype != dtype:
        raise ValueError("Buffer dtype mismatch, expected '%s' but got '%s'" % (cname, x.dtype))
    if x.dim() != ndim:
        raise ValueError("Buffer has wrong number of dimensions (expected %d, got %d)" % (ndim, x.dim()))
    if x.device != torch.device("cuda", device):
        raise ValueError("tensor is on %s, the CRF on cuda:%d" % (x.device, device))
    return x


class SimpleCRFFrame(object):
    """== csimple_crf.SimpleCRFFrame: a handle on one frame of `parent_crf` (which it keeps alive)."""

    def __init__(self, parent_crf, time):
        self._parent = parent_crf
        self._time = time

    @property
    def parent_crf(self):
        return self._parent

    @property
    def time(self):
        self._alive()
        return self._time

    @property
    def num_nodes(self):
        return self._parent._N

    @property
    def num_classes(self):
        return self._parent._C

    @property
    def space_size(self):
        return self._parent._C * self._parent._N

    def _alive(self):
        p = self._parent
        if not (p.first_time <= self._time <= p.last_time) or p.first_time < 0:
            raise IndexError("Time out of range")

    def _call(self, name, *args):
        p = self._parent
        with p.lock:
            _check(getattr(_L(), "fslic_b200_crf_" + name)(p._h, self._time, *args))

    def _dcall(self, name, *args):
        """A device-feed entry point, on the CRF device's current torch stream."""
        p = self._parent
        with p.lock:
            _check(getattr(_L(), "fslic_b200_crfdev_" + name)(p._h, self._time, *args, p._stream()))

    def _fresh_buffer(self):
        return np.zeros([self.num_classes, self.num_nodes], dtype=np.float32)

    @property
    def unaries(self):
        out = self._fresh_buffer()
        self._call("get_unary", _vp(out))
        return out

    @unaries.setter
    def unaries(self, new_value):
        if _is_cuda(new_value):
            a = self._check_dimension(_device_tensor(new_value, self._parent.device, torch.float32, 2, "float"))
            self._dcall("set_unary", a.contiguous().data_ptr())
            return
        a = self._check_dimension(_buffer(new_value, np.float32, 2, "float"))
        self._call("set_unary", _vp(a))

    def get_yxmrgb(self):
        cl = np.zeros(self.num_nodes, CLUSTER_DTYPE)
        self._call("get_clusters", _vp(cl))
        return [[float(c["y"]), float(c["x"]), int(c["num_members"]), float(c["r"]), float(c["g"]), float(c["b"])]
                for c in cl]

    def set_yxmrgb(self, yxmrgb):
        a = _buffer(yxmrgb, np.int32, 2, "int32_t")
        if self.num_nodes != a.shape[0]:
            raise ValueError("Expected the first dimension of yxmrgb to equal to {}".format(self.num_nodes))
        if 6 != a.shape[1]:
            raise ValueError("Expected the second dimension of yxmrgb to equal to 6")
        cl = np.zeros(self.num_nodes, CLUSTER_DTYPE)
        for col, name in enumerate(("y", "x", "num_members", "r", "g", "b")):
            cl[name] = a[:, col].astype(np.uint32) if name == "num_members" else a[:, col]
        cl["number"] = np.arange(self.num_nodes, dtype=np.int64).astype(np.uint16)
        self._call("set_clusters", _vp(cl))

    def get_connectivity(self):
        N = self.num_nodes
        off = np.zeros(N + 1, np.int32)
        p = self._parent
        with p.lock:
            _check(_L().fslic_b200_crf_get_connectivity(p._h, self._time, _vp(off), None, 0))
            nbr = np.zeros(max(int(off[-1]), 1), np.int32)
            _check(_L().fslic_b200_crf_get_connectivity(p._h, self._time, _vp(off), _vp(nbr), len(nbr)))
        return [nbr[off[i]:off[i + 1]].tolist() for i in range(N)]

    def set_connectivity(self, connectivity):
        from .base_slic import NodeConnectivity
        if isinstance(connectivity, NodeConnectivity):
            counts = np.ascontiguousarray(connectivity._counts, np.int64)
            nb = np.asarray(connectivity._neighbors)
            if len(counts) > self.num_nodes:
                raise ValueError("Expected at most {} adjacency lists".format(self.num_nodes))
            mask = np.arange(nb.shape[1])[None, :] < counts[:, None]
            flat = nb[mask].astype(np.int64)  # row-major: row by row, each in list order
        else:
            if len(connectivity) != self.num_nodes:
                raise ValueError("Expected len(connectivity) to be {}".format(self.num_nodes))
            counts, vals = [], []
            for neighbors in connectivity:
                counts.append(len(neighbors))
                for neighbor in neighbors:
                    v = operator.index(neighbor)
                    if v < 0 or v > 0xFFFFFFFF:  # cdef uint32_t neighbor
                        raise OverflowError("value too large to convert to unsigned int" if v > 0 else
                                            "can't convert negative value to unsigned int")
                    vals.append(v)
            counts = np.array(counts, np.int64)
            flat = np.array(vals, np.int64)
        if ((flat < 0) | (flat >= self.num_nodes)).any():
            raise ValueError("neighbour index out of range: the frame has {} nodes".format(self.num_nodes))
        off = np.zeros(len(counts) + 1, np.int32)
        off[1:] = np.cumsum(counts)
        nbr = np.ascontiguousarray(flat, np.int32) if len(flat) else np.zeros(1, np.int32)
        self._call("set_connectivity", len(counts), _vp(off), _vp(nbr))

    def set_unbiased(self):
        self._call("set_unbiased")

    def set_mask(self, classes, confidence):
        if _is_cuda(classes):  # classes are checked on the device: out of range raises ValueError, nothing changes
            a = _device_tensor(classes, self._parent.device, torch.int32, 1, "int")
            confidence = float(confidence)
            if a.shape[0] != self.num_nodes:
                raise ValueError("The dimension of class array should match the number of nodes {}".format(
                    self.num_nodes))
            self._dcall("set_mask", a.contiguous().data_ptr(), C.c_float(confidence))
            return
        a = _buffer(classes, np.int32, 1, "int")
        confidence = float(confidence)
        if a.shape[0] != self.num_nodes:
            raise ValueError("The dimension of class array should match the number of nodes {}".format(self.num_nodes))
        if ((a < 0) | (a >= self.num_classes)).any():
            raise ValueError("class index out of range: there are {} classes".format(self.num_classes))
        self._call("set_mask", _vp(a), C.c_float(confidence))

    def set_proba(self, proba):
        if _is_cuda(proba):
            a = self._check_dimension(_device_tensor(proba, self._parent.device, torch.float32, 2, "float"))
            self._dcall("set_proba", a.contiguous().data_ptr())
            return
        a = self._check_dimension(_buffer(proba, np.float32, 2, "float"))
        self._call("set_proba", _vp(a))

    def get_inferred(self, out=None):
        """q as a new float32 [C, N] numpy array; or, given a contiguous cuda float32 [C, N] tensor `out`, q copied into
        it on the current stream, and `out` returned."""
        if out is not None:
            if not _is_cuda(out):
                raise ValueError("out must be a cuda float32 tensor of shape [num_classes, num_nodes]")
            self._check_dimension(_device_tensor(out, self._parent.device, torch.float32, 2, "float"))
            if not out.is_contiguous():
                raise ValueError("out must be contiguous")
            self._dcall("get_inferred", out.data_ptr())
            return out
        out = self._fresh_buffer()
        self._call("get_inferred", _vp(out))
        return out

    def reset_inferred(self):
        self._call("reset_inferred")

    def temporal_pairwise_energy(self, node_i, other):
        if not isinstance(other, SimpleCRFFrame):
            raise TypeError("not a crf frame")
        node_i = _c_int(node_i)
        if not 0 <= node_i < self.num_nodes:
            raise ValueError("node number is out of range")
        out = C.c_float()
        p, o = self._parent, other._parent
        first, second = sorted((p, o), key=id)  # one global order: no deadlock with the frames swapped
        with first.lock, second.lock:
            _check(_L().fslic_b200_crf_temporal_pairwise_energy(p._h, self._time, node_i, o._h, other._time,
                                                                C.byref(out)))
        return out.value

    def spatial_pairwise_energy(self, node_i, node_j):
        node_i, node_j = _c_int(node_i), _c_int(node_j)
        if not (0 <= node_i < self.num_nodes and 0 <= node_j < self.num_nodes):
            raise ValueError("node number is out of range")
        out = C.c_float()
        self._call("spatial_pairwise_energy", node_i, node_j, C.byref(out))
        return out.value

    def _check_dimension(self, arr):
        if arr.shape[0] != self.num_classes:
            raise ValueError("The first dimension of array should match the number of classes {}".format(
                self.num_classes))
        if arr.shape[1] != self.num_nodes:
            raise ValueError("The second dimension of array should match the number of nodes {}".format(
                self.num_nodes))
        return arr


def _param_property(name):
    def get(self):
        return getattr(self._params(), name)

    def set(self, value):
        with self.lock:
            p = self._params()
            setattr(p, name, float(value))  # stored as float32, like the reference's `float` setter argument
            _check(_L().fslic_b200_crf_set_params(self._h, C.byref(p)))

    return property(get, set)


class SimpleCRF(object):
    """== csimple_crf.SimpleCRF(num_classes, num_nodes), on CUDA device `device`."""

    def __init__(self, num_classes, num_nodes, *, device=0):
        C_, N = _size_t(num_classes), _size_t(num_nodes)
        if C_ > _INT_MAX or N > _INT_MAX or C_ * N > _INT_MAX:
            raise ValueError("num_classes, num_nodes and num_classes * num_nodes must be < 2^31")
        self.lock = threading.RLock()
        self._h = None
        self._C, self._N = C_, N
        self.device = int(device)
        h = C.c_void_p()
        _check(_L().fslic_b200_crf_create(self.device, C_, N, C.byref(h)))
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None):
            _L().fslic_b200_crf_destroy(self._h)
            self._h = None

    def _params(self):
        p = _Params()
        _check(_L().fslic_b200_crf_get_params(self._h, C.byref(p)))
        return p

    spatial_w = _param_property("spatial_w")
    spatial_srgb = _param_property("spatial_srgb")
    spatial_sxy = _param_property("spatial_sxy")
    temporal_w = _param_property("temporal_w")
    temporal_srgb = _param_property("temporal_srgb")
    spatial_smooth_w = _param_property("spatial_smooth_w")
    spatial_smooth_sxy = _param_property("spatial_smooth_sxy")

    def _times(self):
        f, l, n = C.c_int(), C.c_int(), C.c_int()
        _check(_L().fslic_b200_crf_times(self._h, C.byref(f), C.byref(l), C.byref(n)))
        return f.value, l.value, n.value

    @property
    def first_time(self):
        return self._times()[0]

    @property
    def last_time(self):
        return self._times()[1]

    @property
    def num_frames(self):
        return self._times()[2]

    @property
    def space_size(self):
        return self._C * self._N

    def get_frame(self, time):
        time = _c_int(time)
        first, last, _ = self._times()
        if first < 0 or not first <= time <= last:
            raise IndexError("Time out of range")
        return SimpleCRFFrame(self, time)

    def push_slic_frame(self, slic, knn=None):
        """The reference's push_slic_frame as it is evidently meant: its set_yxmrgb demands int32 while to_yxmrgb
        gives float64, so the reference always raises.  Here the model's rows are truncated to int32 (what set_yxmrgb
        would store), the graph of the last assignment is set and the frame made unbiased."""
        if knn is not None:
            conn = slic.slic_model.get_knn_connectivity(slic.last_assignment, knn)  # raises NotImplementedError
        frame = self.push_frame()
        frame.set_yxmrgb(np.ascontiguousarray(slic.slic_model.to_yxmrgb().astype(np.int32)))
        if knn is None:
            conn = slic.slic_model.get_connectivity(slic.last_assignment)
        frame.set_connectivity(conn)
        frame.set_unbiased()
        return frame

    def push_label_frames(self, labels, clusters):
        """Frames from device tensors: int16 cuda labels [H,W] or [B,H,W] and the uint8 [K,32] / [B,K,32] cluster
        records of the same images, as `iterate_batch(..., return_clusters=True)` returns them.  Frame b equals what
        push_slic_frame gives for a Slic whose last_assignment is labels[b] and whose records are clusters[b]: the
        records truncated to int32 as there, the adjacency graph of labels[b] (labels outside [0, K) ignored) and
        unbiased unaries.  Returns one SimpleCRFFrame for [H,W] labels, a list for [B,H,W].  Enqueued on the CRF
        device's current torch stream.  Unlike push_slic_frame, which pushes a blank frame before it fails on
        K != num_nodes, this checks every argument (ValueError) before anything is pushed."""
        from .graph_batch import graph_chunk
        if not _is_cuda(labels) or not _is_cuda(clusters):
            raise ValueError("labels and clusters must be cuda tensors (push_slic_frame takes host arrays)")
        single = labels.dim() == 2
        _device_tensor(labels, self.device, torch.int16, 2 if single else 3, "int16_t")
        _device_tensor(clusters, self.device, torch.uint8, 2 if single else 3, "uint8_t")
        lab = labels[None] if single else labels
        cl = clusters[None] if single else clusters
        B, H, W = (int(v) for v in lab.shape)
        if tuple(cl.shape) != (B, self._N, 32):
            raise ValueError("clusters must be %s with K = num_nodes, got %s" % (
                (self._N, 32) if single else (B, self._N, 32), tuple(clusters.shape)))
        if H == 0 or W == 0:
            raise ValueError("labels must have at least one pixel")
        if not 1 <= self._N <= 65535:
            raise ValueError("push_label_frames needs 1 <= num_nodes <= 65535, the range of the labels")
        lab, cl = lab.contiguous(), cl.contiguous()
        times = np.zeros(B, np.int32)
        if B:
            L = _L()
            dev = torch.device("cuda", self.device)
            with torch.cuda.device(dev), self.lock:
                chunk = graph_chunk(self._N, B)  # images whose graph scratch stays under GRAPH_SCRATCH_CAP
                nbytes = int(L.fslic_b200_crfdev_push_scratch_bytes(self._N, chunk))
                scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
                for b0 in range(0, B, chunk):
                    n = min(chunk, B - b0)
                    _check(L.fslic_b200_crfdev_push_label_frames(
                        self._h, n, H, W, self._N, lab[b0].data_ptr(), cl[b0].data_ptr(), scratch.data_ptr(), nbytes,
                        self._stream(), times[b0:].ctypes.data_as(C.POINTER(C.c_int))))
        frames = [SimpleCRFFrame(self, int(t)) for t in times]
        return frames[0] if single else frames

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(torch.device("cuda", self.device)).cuda_stream)

    def push_frame(self):
        t = C.c_int()
        with self.lock:
            _check(_L().fslic_b200_crf_push_frame(self._h, C.byref(t)))
        return SimpleCRFFrame(self, t.value)

    def pop_frame(self):
        t = C.c_int()
        with self.lock:
            _check(_L().fslic_b200_crf_pop_frame(self._h, C.byref(t)))
        return t.value

    def initialize(self):
        with self.lock:
            _check(_L().fslic_b200_crf_initialize(self._h))

    def inference(self, max_iter):
        max_iter = _size_t(max_iter)
        with self.lock:
            _check(_L().fslic_b200_crf_inference(self._h, max_iter, None))


class SimpleCRFGroup(object):
    """The SimpleCRFs `crfs` (distinct, with the same num_classes, num_nodes and device) driven together: each call
    runs every member in the same kernel launches, on the device's current torch stream, and leaves every member as
    its own calls would.  Member b takes image b of each batch.  The members keep their whole surface; the group holds
    no state of its own besides the list."""

    def __init__(self, crfs):
        crfs = list(crfs)
        if not crfs:
            raise ValueError("a SimpleCRFGroup needs at least one SimpleCRF")
        if not all(isinstance(c, SimpleCRF) for c in crfs):
            raise ValueError("every member must be a SimpleCRF")
        if len(set(map(id, crfs))) != len(crfs):
            raise ValueError("a SimpleCRF is in the group twice")
        c0 = crfs[0]
        if any((c._C, c._N, c.device) != (c0._C, c0._N, c0.device) for c in crfs):
            raise ValueError("members differ in num_classes, num_nodes or device")
        self._crfs = crfs
        self._handles = (C.c_void_p * len(crfs))(*[c._h.value for c in crfs])
        self._locks = [c.lock for c in sorted(crfs, key=id)]  # one global order, as temporal_pairwise_energy takes it

    def _stream(self):
        return self._crfs[0]._stream()

    @property
    def crfs(self):
        return list(self._crfs)

    def __len__(self):
        return len(self._crfs)

    @contextlib.contextmanager
    def _locked(self):
        """The members' device current and all their locks held."""
        with contextlib.ExitStack() as stack:
            stack.enter_context(torch.cuda.device(torch.device("cuda", self._crfs[0].device)))
            for lock in self._locks:
                stack.enter_context(lock)
            yield

    def _call(self, name, *args, first=0, count=None):
        """fslic_b200_<name> over members first .. first + count - 1 (default: all), under _locked()."""
        n = len(self._crfs) - first if count is None else count
        handles = C.c_void_p(C.addressof(self._handles) + first * C.sizeof(C.c_void_p))
        with self._locked():
            _check(getattr(_L(), "fslic_b200_" + name)(handles, n, *args))

    def _group_tensor(self, x, cname="float"):
        c0 = self._crfs[0]
        _device_tensor(x, c0.device, torch.float32, 3, cname)
        want = (len(self._crfs), c0._C, c0._N)
        if tuple(x.shape) != want:
            raise ValueError("expected a tensor of shape %s, got %s" % (want, tuple(x.shape)))
        return x

    def push_label_frames(self, labels, clusters):
        """Frame b from int16 cuda labels[b] ([B,H,W]) and uint8 cuda records clusters[b] ([B,K,32]), B = len(group),
        appended to member b: what member b's own push_label_frames(labels[b], clusters[b]) gives.  Every argument is
        checked (ValueError) before anything is pushed.  Returns the new SimpleCRFFrame of each member."""
        from .graph_batch import graph_chunk
        if not _is_cuda(labels) or not _is_cuda(clusters):
            raise ValueError("labels and clusters must be cuda tensors")
        c0 = self._crfs[0]
        B, K = len(self._crfs), c0._N
        _device_tensor(labels, c0.device, torch.int16, 3, "int16_t")
        _device_tensor(clusters, c0.device, torch.uint8, 3, "uint8_t")
        if labels.shape[0] != B or tuple(clusters.shape) != (B, K, 32):
            raise ValueError("labels must be [%d,H,W] and clusters [%d,%d,32], got %s and %s" % (
                B, B, K, tuple(labels.shape), tuple(clusters.shape)))
        H, W = int(labels.shape[1]), int(labels.shape[2])
        if H == 0 or W == 0:
            raise ValueError("labels must have at least one pixel")
        if not 1 <= K <= 65535:
            raise ValueError("push_label_frames needs 1 <= num_nodes <= 65535, the range of the labels")
        lab, cl = labels.contiguous(), clusters.contiguous()
        times = np.zeros(B, np.int32)
        with self._locked():
            chunk = graph_chunk(K, B)  # images whose graph scratch stays under GRAPH_SCRATCH_CAP
            nbytes = int(_L().fslic_b200_crfdev_push_scratch_bytes(K, chunk))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=torch.device("cuda", c0.device))
            for b0 in range(0, B, chunk):
                self._call("crfdev_group_push_label_frames", H, W, K, lab[b0].data_ptr(), cl[b0].data_ptr(),
                           scratch.data_ptr(), nbytes, c0._stream(), times[b0:].ctypes.data_as(C.POINTER(C.c_int)),
                           first=b0, count=min(chunk, B - b0))
        return [SimpleCRFFrame(c, int(t)) for c, t in zip(self._crfs, times)]

    def set_proba(self, proba):
        """set_proba of each member's newest frame from float32 cuda proba [B, C, N] (-logf(p))."""
        self._call("crfdev_group_set_proba", self._group_tensor(proba).contiguous().data_ptr(), self._stream())

    def reset_inferred(self):
        """reset_inferred of each member's newest frame."""
        self._call("crfdev_group_reset_inferred", self._stream())

    def inference(self, max_iter):
        """max_iter mean-field steps of every member, asynchronously."""
        self._call("crfgroup_inference", _size_t(max_iter), self._stream())

    def get_inferred(self, out=None):
        """q of each member's newest frame into the contiguous float32 cuda tensor `out` [B, C, N] (a new one if None),
        enqueued on the current stream; returns it."""
        c0 = self._crfs[0]
        if out is None:
            out = torch.empty((len(self._crfs), c0._C, c0._N), dtype=torch.float32,
                              device=torch.device("cuda", c0.device))
        if not _is_cuda(out):
            raise ValueError("out must be a cuda float32 tensor of shape [len(group), num_classes, num_nodes]")
        self._group_tensor(out)
        if not out.is_contiguous():
            raise ValueError("out must be contiguous")
        self._call("crfdev_group_get_inferred", out.data_ptr(), self._stream())
        return out

    def pop_frame(self):
        """pop_frame of every member; the popped times, -1 for a member that had no frames."""
        times = np.zeros(len(self._crfs), np.int32)
        self._call("crfgroup_pop_frame", times.ctypes.data_as(C.POINTER(C.c_int)))
        return times.tolist()
