"""LSC (linear spectral clustering) on the GPU against its CPU checker -- the compiled, unmodified reference's ContextLSC
with num_threads=1 (oracle_lsc/_ref) where it was built, else the restatement the CPU suite pins to the reference's
digests --: labels, pre-CCA labels, raw Cluster bytes and the before_iteration stage buffers, tolerance 0."""
import numpy as np
import pytest
import torch

from class_checks import LSC, assert_kernel
from lsc_cases import LSC_BIG_CASE, LSC_CASES, LSC_SWEEP_CASES, lsc_args, lsc_image

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lsc_checker():
    from oracle_lsc.lsc import Port, Ref
    return Ref() if Ref.available() else Port()


def _gpu_engine(H, W, K, B=1):
    from fast_slic_b200 import get_engine
    return get_engine(H, W, K, B, 0)


def _stages_equal(name, r, eng, st, b=0):
    means, weights, cinit = [x[b].cpu().numpy() for x in eng.debug_lsc_stages(b + 1)]
    assert means.view(np.uint32).tolist() == st["means"].view(np.uint32).tolist(), "%s round %d: means differ" % (name, r)
    bad = int((weights.view(np.uint32) != st["weights"].view(np.uint32)).sum())
    assert bad == 0, "%s round %d: %d weights differ" % (name, r, bad)
    bad = int((cinit.view(np.uint32) != st["cinit"].view(np.uint32)).sum())
    assert bad == 0, "%s round %d: %d initial centroid features differ" % (name, r, bad)


def _compare(lsc_checker, case, manhattan=True):
    name = case[0]
    img, K, a = lsc_image(case)
    H, W, _ = img.shape
    eng = _gpu_engine(H, W, K)
    t = torch.from_numpy(img).cuda()[None].contiguous()
    cl_gpu = eng.initialize_clusters(t)
    cl = lsc_checker.initialize(img, K)
    assert cl_gpu.cpu().numpy().tobytes() == cl.tobytes(), name + ": initialize_clusters differs"
    p = eng.params(a["compactness"], a["min_size_factor"], a["subsample_stride"], a["convert_to_lab"], a["max_iter"])
    for r in range(2):  # cold, then warm on the records the first call left
        lab = eng.iterate_lsc(t, cl_gpu, p, manhattan_spatial_dist=manhattan)[0].cpu().numpy().view(np.uint16)
        _, pre = eng.debug_stages(1)
        pre = pre[0].cpu().numpy().view(np.uint16)
        want, st = lsc_checker.iterate_lsc(img, cl, *lsc_args(a), stages=True)
        assert (pre == st["pre"]).all(), "%s round %d: pre-CCA labels differ (%d px)" % (name, r, int((pre != st["pre"]).sum()))
        assert (lab == want).all(), "%s round %d: labels differ (%d px)" % (name, r, int((lab != want).sum()))
        assert cl_gpu[0].cpu().numpy().tobytes() == cl.tobytes(), "%s round %d: Cluster bytes differ" % (name, r)
        _stages_equal(name, r, eng, st)
        assert_kernel("%s round %d" % (name, r), eng.dispatch(), LSC, a["max_iter"])


ENGINE_CASES = LSC_CASES + [LSC_BIG_CASE] + LSC_SWEEP_CASES


@pytest.mark.parametrize("case", ENGINE_CASES, ids=[c[0] for c in ENGINE_CASES])
def test_lsc_engine_matches_checker(lsc_checker, case):
    """The hand-picked cases, the bench's shape and the seeded sweep (lsc_cases.py::lsc_sweep_case): every stage of both
    calls, on k_assign_lsc."""
    _compare(lsc_checker, case)


def test_lsc_manhattan_flag_has_no_effect(lsc_checker):
    """ContextLSC never reads the spatial patch: manhattan_spatial_dist=False gives the same bits."""
    for case in LSC_CASES[:3]:
        _compare(lsc_checker, case, manhattan=False)


def test_lsc_class_iterate_matches_checker(lsc_checker):
    """fast_slic_b200.LSC(num_threads=1).iterate, cold then warm: int16 labels and the model's Cluster records."""
    import fast_slic_b200 as fs
    for case in (LSC_CASES[0], LSC_CASES[2], LSC_CASES[3]):
        img, K, a = lsc_image(case)
        s = fs.LSC(num_components=K, compactness=a["compactness"], min_size_factor=a["min_size_factor"],
                   subsample_stride=a["subsample_stride"], convert_to_lab=a["convert_to_lab"], num_threads=1)
        cl = lsc_checker.initialize(img, K)
        for r in range(2):
            got = s.iterate(img, max_iter=a["max_iter"])
            want = lsc_checker.iterate_lsc(img, cl, *lsc_args(a))
            assert got.dtype == np.int16 and (got.view(np.uint16) == want).all(), "%s round %d" % (case[0], r)
            assert s.slic_model.cluster_array.tobytes() == cl.tobytes(), "%s round %d: clusters" % (case[0], r)
        import json
        tree = json.loads(s.slic_model.last_timing_report)
        assert [c["name"] for c in tree["children"]] == ["cielab_conversion", "before_iteration", "assign", "update",
                                                         "after_update", "full_assign", "enforce_connectivity"]


@pytest.mark.parametrize("on_device", [False, True], ids=["host", "device"])
def test_lsc_iterate_batch_matches_checker(lsc_checker, on_device):
    """iterate_batch with B = 3 different images, numpy and cuda-tensor inputs: each image equals its own single run."""
    import fast_slic_b200 as fs
    from cases import make_image
    H, W, K = 96, 124, 40
    imgs = np.stack([make_image(kind, H, W, seed=70 + b) for b, kind in enumerate(("syn", "noise", "blocks"))])
    s = fs.LSC(num_components=K, num_threads=1)
    src = torch.from_numpy(imgs).cuda().contiguous() if on_device else imgs
    labels, clusters = s.iterate_batch(src, max_iter=10, return_clusters=True)
    if on_device:
        labels = labels.cpu().numpy()
        clusters = clusters.cpu().numpy().view(fs.SlicModel(1).cluster_array.dtype).reshape(3, K)
    for b in range(3):
        cl = lsc_checker.initialize(imgs[b], K)
        want, st = lsc_checker.iterate_lsc(imgs[b], cl, 10, 10.0, 0.25, 3, True, stages=True)
        assert (labels[b].view(np.uint16) == want).all(), "image %d: labels differ" % b
        assert clusters[b].tobytes() == cl.tobytes(), "image %d: Cluster bytes differ" % b
