"""SimpleCRF on a non-blocking CUDA stream, and the conversion rules of the frame methods.

Every copy and kernel of a CRF goes to the stream last passed to fslic_b200_crf_inference.  Here that stream is a
PyTorch side stream (created cudaStreamNonBlocking, so nothing orders it with the legacy default stream): the cases
must still be bit-identical to the checker, and each query must see the work enqueued before it."""
import ctypes as C
import os

import numpy as np
import pytest

from crf_cases import CRF_CASES, nan_class_equal, run_case
from test_crf_gpu import Gpu

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


class GpuSideStream(Gpu):
    """inference() on a non-blocking side stream; every later call runs on that stream too."""

    def __init__(self, C_, N):
        import torch
        super().__init__(C_, N)
        self.stream = torch.cuda.Stream(device=0)

    def inference(self, k):
        from fast_slic_b200 import crf as crf_mod
        with self.crf.lock:
            crf_mod._check(crf_mod._L().fslic_b200_crf_inference(self.crf._h, k, C.c_void_p(self.stream.cuda_stream)))


@pytest.mark.parametrize("name", ["c3_n100_t3_popush", "c3_n100_t3_params", "c21_n1600_t5_slic", "c3_n100_t3_raw_nan"])
def test_case_on_a_non_blocking_stream(name):
    from oracle_crf.crf import Port, Ref
    case = {c[0]: c for c in CRF_CASES}[name]
    chk = Ref if os.path.exists(os.path.join(ROOT, "oracle_crf", "_ref", "libfslic_ref_crf.so")) else Port
    model, ref = GpuSideStream(case[1], case[2]), chk(case[1], case[2])
    for m in (model, ref):  # one blank frame and one iteration: from here on the CRF works on the side stream
        m.push()
        m.inference(1)
        m.pop()
    got = run_case(model, case)
    want = run_case(ref, case)
    assert set(got) == set(want)
    bad = sorted(k for k in got if not nan_class_equal(got[k], want[k]))
    assert not bad, bad[:8]


def test_queries_follow_the_side_stream():
    """An energy query right after a params change and a long inference on the side stream sees the new params."""
    import torch
    from fast_slic_b200.crf import SimpleCRF
    crf = SimpleCRF(21, 2000)
    side = torch.cuda.Stream(device=0)
    from fast_slic_b200 import crf as crf_mod
    rng = np.random.RandomState(3)
    frames = [crf.push_frame() for _ in range(3)]
    for f in frames:
        y = np.stack([rng.randint(0, 720, 2000), rng.randint(0, 1280, 2000), rng.randint(1, 50, 2000)] +
                     [rng.randint(0, 256, 2000) for _ in range(3)], 1).astype(np.int32)
        f.set_yxmrgb(y)
        f.set_connectivity([rng.randint(0, 2000, 8).tolist() for _ in range(2000)])
        f.set_unbiased()
    crf.initialize()
    values = []
    for w in (1.0, 2.0, 3.0):
        crf.spatial_w = w
        with crf.lock:
            crf_mod._check(crf_mod._L().fslic_b200_crf_inference(crf._h, 50, C.c_void_p(side.cuda_stream)))
        values.append(frames[1].spatial_pairwise_energy(0, 1))
    e = np.float32(values[0])
    assert e > 0
    assert values[1] == 2 * e and values[2] == np.float32(3) * e  # spatial_w * expf(...) with smooth_w = 0
    assert np.isfinite(frames[1].get_inferred()).all()


def test_frame_arguments_convert_like_cython():
    from fast_slic_b200.crf import SimpleCRF
    crf = SimpleCRF(3, 3)
    frame = crf.push_frame()
    for bad in ([[None], [], []], [[1.0], [], []], [["1"], [], []]):
        with pytest.raises(TypeError):
            frame.set_connectivity(bad)
    with pytest.raises(TypeError):
        frame.spatial_pairwise_energy(0.0, 1)
    with pytest.raises(OverflowError):
        frame.spatial_pairwise_energy(2 ** 31, 1)
    with pytest.raises(TypeError):
        crf.get_frame(0.0)
    with pytest.raises(OverflowError):
        crf.inference(2 ** 64)
    with pytest.raises(TypeError):
        crf.inference(1.0)
    frame.set_connectivity([[np.int64(1)], [np.uint32(2)], []])
    assert frame.get_connectivity() == [[1], [2], []]


def test_temporal_energy_across_two_crfs_from_two_threads():
    """Both CRFs' locks are taken in one global order, so swapped frames on two threads cannot deadlock."""
    import threading
    from fast_slic_b200.crf import SimpleCRF
    a, b = SimpleCRF(2, 4), SimpleCRF(2, 4)
    fa, fb = a.push_frame(), b.push_frame()
    fb.set_yxmrgb(np.array([[0, 0, 1, 9, 9, 9]] * 4, np.int32))
    errors = []

    def run(x, y):
        try:
            for _ in range(200):
                x.temporal_pairwise_energy(1, y)
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=run, args=(fa, fb)), threading.Thread(target=run, args=(fb, fa))]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=60)
    assert not any(t.is_alive() for t in ts) and not errors
    assert fa.temporal_pairwise_energy(1, fb) == fb.temporal_pairwise_energy(1, fa) > 0
