"""SimpleCRF on the GPU (fast_slic_b200.crf): the reference's own CRF tests, every seeded case against the checker
(the compiled reference where it was built, else the restatement the CPU suite pins to its digests) at tolerance 0,
push_slic_frame end to end, the device expf clone on every input, and the refusal rules."""
import ctypes as C
import hashlib
import os
import gc

import numpy as np
import pytest

from crf_cases import CRF_CASES, GPU_BIG_CASE, nan_class_equal, run_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "crf_reference_digests.npz")


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def SimpleCRF(*a, **k):
    from fast_slic_b200.crf import SimpleCRF as S
    return S(*a, **k)


class Gpu:
    """fast_slic_b200.crf behind the oracle_crf surface (tests/crf_cases.py)."""

    def __init__(self, C_, N):
        self.crf = SimpleCRF(C_, N)
        self.N = N

    def set_params(self, **kw):
        for k, v in kw.items():
            setattr(self.crf, k, v)

    def push(self):
        return self.crf.push_frame().time

    def pop(self):
        return self.crf.pop_frame()

    def first(self):
        return self.crf.first_time

    def last(self):
        return self.crf.last_time

    def f(self, t):
        return self.crf.get_frame(t)

    def set_clusters(self, t, cl):
        y = np.stack([cl[n].astype(np.int64) for n in ("y", "x", "num_members", "r", "g", "b")], 1)
        self.f(t).set_yxmrgb(np.ascontiguousarray(y.astype(np.uint32).view(np.int32)))

    def set_connectivity(self, t, off, nbr):
        self.f(t).set_connectivity([nbr[off[i]:off[i + 1]].tolist() for i in range(self.N)])

    def set_unary(self, t, u):
        self.f(t).unaries = u

    def get_unary(self, t):
        return self.f(t).unaries

    def set_unbiased(self, t):
        self.f(t).set_unbiased()

    def set_mask(self, t, cls, conf):
        self.f(t).set_mask(cls, conf)

    def set_proba(self, t, p):
        self.f(t).set_proba(p)

    def get_inferred(self, t):
        return self.f(t).get_inferred()

    def reset_inferred(self, t):
        self.f(t).reset_inferred()

    def initialize(self):
        self.crf.initialize()

    def inference(self, k):
        self.crf.inference(k)

    def spatial(self, t, i, j):
        return np.float32(self.f(t).spatial_pairwise_energy(i, j))

    def temporal(self, t, i, other):
        return np.float32(self.f(t).temporal_pairwise_energy(i, self.f(other)))


@pytest.fixture(scope="module")
def checker_cls():
    from oracle_crf.crf import Port, Ref
    return Ref if os.path.exists(os.path.join(ROOT, "oracle_crf", "_ref", "libfslic_ref_crf.so")) else Port


def _compare(got, want, name):
    assert set(got) == set(want)
    bad = sorted(k for k in got if not nan_class_equal(got[k], want[k]))
    assert not bad, "%s: %s differ from the checker" % (name, bad[:8])


@pytest.mark.parametrize("case", CRF_CASES, ids=[c[0] for c in CRF_CASES])
def test_case_bit_identical_to_checker(checker_cls, case):
    """Unaries, q after initialize() and every inference(), and the pairwise energies, at tolerance 0 (any NaN equals
    any NaN at the same position: x86 and the GPU make different NaN payloads)."""
    got = run_case(Gpu(case[1], case[2]), case)
    want = run_case(checker_cls(case[1], case[2]), case)
    _compare(got, want, case[0])


def test_big_case(checker_cls):
    case = GPU_BIG_CASE
    got = run_case(Gpu(case[1], case[2]), case, energies=False)
    want = run_case(checker_cls(case[1], case[2]), case, energies=False)
    _compare(got, want, case[0])


def test_push_slic_frame_end_to_end(checker_cls):
    """Slic on three synthetic frames with warm start; each frame pushed with push_slic_frame, then set_proba,
    initialize and inference, against the checker fed the same clusters and graph."""
    from fast_slic_b200 import Slic
    from oracle.oracle import CLUSTER_DTYPE, synthetic_image
    K, Cc = 300, 4
    slic = Slic(num_components=K)
    crf = SimpleCRF(Cc, K)
    chk = checker_cls(Cc, K)
    rng = np.random.RandomState(7)
    for t in range(3):
        slic.iterate(synthetic_image(240, 320, seed=30 + t))
        frame = crf.push_slic_frame(slic)
        y = slic.slic_model.to_yxmrgb().astype(np.int32)
        cl = np.zeros(K, CLUSTER_DTYPE)
        for col, n in enumerate(("y", "x", "num_members", "r", "g", "b")):
            cl[n] = y[:, col].astype(np.uint32) if n == "num_members" else y[:, col]
        lists = slic.slic_model.get_connectivity(slic.last_assignment).tolist()
        assert frame.get_connectivity() == lists
        assert frame.get_yxmrgb() == y.tolist()
        tc = chk.push()
        chk.set_clusters(tc, cl)
        off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
        chk.set_connectivity(tc, off, np.array([j for x in lists for j in x], np.int32))
        chk.set_unbiased(tc)
        assert nan_class_equal(frame.unaries, chk.get_unary(tc))
        p = rng.dirichlet(np.ones(Cc), K).T.astype(np.float32).copy()
        frame.set_proba(p)
        chk.set_proba(tc, p)
    crf.initialize()
    chk.initialize()
    crf.inference(5)
    chk.inference(5)
    for t in range(3):
        assert nan_class_equal(crf.get_frame(t).get_inferred(), chk.get_inferred(t))
    with pytest.raises(NotImplementedError):
        crf.push_slic_frame(slic, knn=4)


def test_device_expf_clone_on_every_input():
    import torch
    from fast_slic_b200 import crf as crf_mod
    L = crf_mod._L()
    z = np.load(REF_DIGESTS)
    want = bytes(z["sha"][z["keys"].tolist().index("expf/all")])
    chunk = 1 << 28
    buf = torch.empty(chunk, dtype=torch.float32, device="cuda:0")
    host = torch.empty(chunk, dtype=torch.float32, pin_memory=True)
    h = hashlib.sha256()
    for first in range(0, 1 << 32, chunk):
        st = torch.cuda.current_stream(0)
        assert L.fslic_b200_debug_expf_device(0, first, chunk, C.c_void_p(buf.data_ptr()), C.c_void_p(st.cuda_stream)) == 0
        host.copy_(buf)
        h.update(host.numpy().tobytes())
    assert h.digest() == want


# ---- the reference's test/test_crf.py, against fast_slic_b200.crf

def test_crf_basic():
    crf = SimpleCRF(3, 100)
    assert crf.space_size == 300
    assert crf.first_time == -1
    assert crf.last_time == -1
    assert crf.num_frames == 0
    with pytest.raises(IndexError):
        crf.get_frame(10)
    assert crf.pop_frame() == -1


def test_crf_frame():
    crf = SimpleCRF(3, 100)
    frame = crf.push_frame()
    assert crf.num_frames == 1
    assert crf.first_time == frame.time
    assert crf.last_time == frame.time
    assert frame.space_size == 300
    assert frame.time == 0
    assert crf.get_frame(0).time == 0


def test_crf_frame_2():
    crf = SimpleCRF(3, 100)
    frame_1 = crf.push_frame()
    frame_2 = crf.push_frame()
    assert crf.num_frames == 2
    assert crf.first_time == frame_1.time
    assert crf.last_time == frame_2.time
    assert crf.pop_frame() == 0
    assert crf.first_time == crf.last_time == 1


def test_gc():
    crf = SimpleCRF(3, 100)
    frame = crf.push_frame()
    del crf
    gc.collect()
    frame.unaries
    frame.get_inferred()


def test_unaries():
    crf = SimpleCRF(3, 3)
    frame = crf.push_frame()
    frame.set_unbiased()
    # the reference compares with np.log(3) under NumPy 1's value-based casting; NumPy 2 compares in float64
    assert (frame.unaries == np.float32(np.log(3))).all()
    frame.set_mask(np.array([0, 1, 2], np.int32), 0.5)
    exp_unaries = -np.log(np.array([[2 / 3., 1 / 6., 1 / 6.], [1 / 6., 2 / 3., 1 / 6.], [1 / 6., 1 / 6., 2 / 3.]]))
    assert np.isclose(frame.unaries, exp_unaries).all()
    prob = np.array([[0.7, 0.5, 0.1], [0.1, 0.3, 0.15], [0.2, 0.2, 0.75]], np.float32)
    frame.set_proba(prob)
    assert np.isclose(frame.unaries, -np.log(prob)).all()


def test_proba():
    crf = SimpleCRF(3, 3)
    frame = crf.push_frame()
    prob = np.array([[0.7, 0.5, 0.1], [0.1, 0.3, 0.15], [0.2, 0.2, 0.75]], np.float32)
    frame.set_proba(prob)
    assert np.isclose(frame.get_inferred(), 0).all()
    crf.initialize()
    assert np.isclose(frame.get_inferred(), prob).all()


def test_initial_inferred():
    crf = SimpleCRF(3, 3)
    frame = crf.push_frame()
    frame.set_unbiased()
    assert (frame.get_inferred() == 0).all()
    frame.reset_inferred()
    assert np.isclose(frame.get_inferred(), 1 / 3.).all()


def test_set_yxmrgb():
    crf = SimpleCRF(3, 3)
    frame = crf.push_frame()
    frame.set_yxmrgb(np.array([[1, 2, 1, 3, 4, 5], [6, 7, 2, 8, 9, 10], [11, 12, 3, 13, 14, 15]], np.int32))
    res = frame.get_yxmrgb()
    assert len(res) == 3
    assert res[0] == [1, 2, 1, 3, 4, 5]
    assert res[1] == [6, 7, 2, 8, 9, 10]
    assert res[2] == [11, 12, 3, 13, 14, 15]


def test_set_connectivity():
    crf = SimpleCRF(3, 3)
    frame = crf.push_frame()
    assert frame.get_connectivity() == [[], [], []]
    with pytest.raises(TypeError):
        frame.set_connectivity([None, None, None])
    frame.set_connectivity([[0, 1], [2], [0]])
    assert frame.get_connectivity() == [[0, 1], [2], [0]]


def test_spatial_energy():
    spatial_srgb, spatial_w, spatial_sxy = 3.5, 1.9, 2.4
    crf = SimpleCRF(3, 2)
    crf.spatial_srgb = spatial_srgb
    crf.spatial_w = spatial_w
    crf.spatial_sxy = spatial_sxy
    assert np.isclose(crf.spatial_srgb, spatial_srgb)
    assert np.isclose(crf.spatial_w, spatial_w)
    assert np.isclose(crf.spatial_sxy, spatial_sxy)
    frame = crf.push_frame()
    frame.set_yxmrgb(np.array([[1, 1, 1, 1, 2, 6], [0, 0, 1, 4, 5, 3]], np.int32))
    energy = spatial_w * np.exp(-((1 - 4) ** 2 + (2 - 5) ** 2 + (6 - 3) ** 2) / (2 * spatial_srgb ** 2) -
                                ((1 - 0) ** 2 + (1 - 0) ** 2) / (2 * spatial_sxy ** 2))
    assert np.isclose(frame.spatial_pairwise_energy(0, 1), energy)
    assert np.isclose(frame.spatial_pairwise_energy(1, 0), energy)
    assert np.isclose(frame.spatial_pairwise_energy(0, 0), 0)
    assert np.isclose(frame.spatial_pairwise_energy(1, 1), 0)


def test_temporal_energy():
    temporal_srgb, temporal_w = 3.5, 1.9
    crf = SimpleCRF(3, 1)
    crf.temporal_srgb = temporal_srgb
    crf.temporal_w = temporal_w
    assert np.isclose(crf.temporal_srgb, temporal_srgb)
    assert np.isclose(crf.temporal_w, temporal_w)
    frame_1 = crf.push_frame()
    frame_2 = crf.push_frame()
    frame_1.set_yxmrgb(np.array([[0, 0, 1, 1, 2, 6]], np.int32))
    frame_2.set_yxmrgb(np.array([[0, 0, 1, 4, 5, 3]], np.int32))
    energy = temporal_w * np.exp(-(((1 - 4) ** 2 + (2 - 5) ** 2 + (6 - 3) ** 2) / (2 * temporal_srgb ** 2)))
    assert np.isclose(frame_1.temporal_pairwise_energy(0, frame_2), energy)
    assert np.isclose(frame_2.temporal_pairwise_energy(0, frame_1), energy)
    assert np.isclose(frame_1.temporal_pairwise_energy(0, frame_1), 0)
    assert np.isclose(frame_2.temporal_pairwise_energy(0, frame_2), 0)


# ---- validation and the decisions where the reference is undefined

def test_params_store_float32():
    crf = SimpleCRF(2, 2)
    assert (crf.spatial_w, crf.temporal_w, crf.spatial_srgb, crf.temporal_srgb, crf.spatial_sxy, crf.spatial_smooth_w,
            crf.spatial_smooth_sxy) == (10, 10, 13, 13, 80, 0, 3)
    crf.spatial_w = 1.9
    assert crf.spatial_w == float(np.float32(1.9)) != 1.9


def test_out_of_range_refusals_leave_state_untouched():
    crf = SimpleCRF(3, 3)
    frame = crf.push_frame()
    frame.set_connectivity([[1], [2], [0]])
    for bad in ([[3], [], []], [[0], [2 ** 31], []]):
        with pytest.raises(ValueError):
            frame.set_connectivity(bad)
    for bad in ([[-1], [], []], [[2 ** 32], [], []]):
        with pytest.raises(OverflowError):
            frame.set_connectivity(bad)
    assert frame.get_connectivity() == [[1], [2], [0]]
    with pytest.raises(ValueError):
        frame.set_connectivity([[0]])
    frame.set_unbiased()
    for cls in ([0, 1, 3], [0, -1, 2]):
        with pytest.raises(ValueError):
            frame.set_mask(np.array(cls, np.int32), 0.5)
    assert (frame.unaries == np.float32(np.log(3))).all()
    with pytest.raises(ValueError):
        frame.spatial_pairwise_energy(0, 3)
    with pytest.raises(ValueError):
        frame.temporal_pairwise_energy(-1, frame)
    with pytest.raises(TypeError):
        frame.temporal_pairwise_energy(0, None)


def test_memoryview_rules():
    crf = SimpleCRF(2, 3)
    frame = crf.push_frame()
    with pytest.raises(ValueError, match="dtype mismatch"):
        frame.set_proba(np.ones((2, 3)))
    with pytest.raises(ValueError, match="wrong number of dimensions"):
        frame.set_proba(np.ones(6, np.float32))
    with pytest.raises(ValueError, match="C-contiguous"):
        frame.set_proba(np.ones((3, 2), np.float32).T)
    with pytest.raises(ValueError, match="first dimension"):
        frame.unaries = np.ones((3, 3), np.float32)
    with pytest.raises(ValueError, match="second dimension"):
        frame.set_proba(np.ones((2, 2), np.float32))
    with pytest.raises(ValueError, match="number of nodes"):
        frame.set_mask(np.zeros(2, np.int32), 0.5)
    with pytest.raises(ValueError, match="dtype mismatch"):
        frame.set_yxmrgb(np.zeros((3, 6), np.int64))
    with pytest.raises(ValueError, match="second dimension of yxmrgb"):
        frame.set_yxmrgb(np.zeros((3, 5), np.int32))
    with pytest.raises(ValueError, match="len\\(connectivity\\)"):
        frame.set_connectivity([[], []])


def test_popped_frame_handle_raises_index_error():
    crf = SimpleCRF(2, 3)
    frame = crf.push_frame()
    crf.push_frame()
    assert crf.pop_frame() == 0
    with pytest.raises(IndexError):
        frame.get_inferred()
    with pytest.raises(IndexError):
        frame.set_unbiased()
    with pytest.raises(IndexError):
        crf.get_frame(0)


def test_empty_shapes_and_empty_crf():
    for C_, N in ((0, 4), (3, 0), (0, 0)):
        crf = SimpleCRF(C_, N)
        frame = crf.push_frame()
        frame.set_unbiased()
        crf.initialize()
        crf.inference(2)
        assert frame.get_inferred().shape == (C_, N)
    crf = SimpleCRF(2, 2)
    crf.inference(0)
    with pytest.raises(IndexError):
        crf.inference(1)
    with pytest.raises(OverflowError):
        crf.inference(-1)
