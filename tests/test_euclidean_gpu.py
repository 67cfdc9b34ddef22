"""manhattan_spatial_dist=False on the GPU: every CUDA path against the Euclidean checker (the compiled reference where
it was built, else the restatement the CPU suite pins to the reference's digests), labels and raw Cluster bytes,
tolerance 0."""
import numpy as np
import pytest
import torch

from cases import make_image, split_kwargs, sweep_case_id
from euclid_cases import (EUCLID_CASES, EUCLID_PREEMPT_CASES, EUCLID_PREEMPT_SWEEP, EUCLID_REAL_CASES, EUCLID_REAL_SWEEP,
                          EUCLID_SAME_CASES, EUCLID_WARM_CASE, case_id, preempt_case_id, preempt_sweep_id)
from class_checks import PREEMPT, check_class_call

pytestmark = pytest.mark.gpu

AS_LIST = 32  # candidate capacity of one warp tile of the assign kernels (assign.cuh)


class Euclid:
    """What the tests compare against: the compiled, unmodified reference run with manhattan_spatial_dist=False
    (oracle_euclid/_ref, SlicAvx2 path) where it was built, else the plain-C restatement that the CPU suite pins to the
    reference's outputs (tests/golden/euclid_reference_digests.npz).  `manhattan=True` calls go to the session checker."""

    def __init__(self, checker):
        from oracle_euclid.euclid import Port, Ref
        self.c = checker
        self.kind = "reference" if Ref.available() else "port"
        self._impl = Ref() if self.kind == "reference" else Port()
        self._kw = dict(arch="x64/avx2", num_threads=checker._threads) if self.kind == "reference" else {}

    def initialize(self, image, K):
        return self.c.initialize(image, K)

    def iterate(self, image, clusters, max_iter=10, compactness=10.0, min_size_factor=0.25, stride=3, convert_to_lab=True,
                stages=False, preemptive=False, preemptive_thres=0.05, manhattan=False):
        if manhattan:
            return self.c.iterate(image, clusters, max_iter, compactness, min_size_factor, stride, convert_to_lab,
                                  stages=stages, preemptive=preemptive, preemptive_thres=preemptive_thres)
        return self._impl.iterate(image, clusters, max_iter, compactness, min_size_factor, stride, convert_to_lab,
                                  stages=stages, preemptive=preemptive, preemptive_thres=preemptive_thres, **self._kw)

    def iterate_real(self, variant, image, clusters, max_iter=10, compactness=10.0, min_size_factor=0.25, stride=3,
                     convert_to_lab=True, stages=False):
        return self._impl.iterate_real(variant, image, clusters, max_iter, compactness, min_size_factor, stride,
                                       convert_to_lab, stages=stages)


@pytest.fixture(scope="module")
def euclid(checker):
    return Euclid(checker)


def _args(a):
    return (a["max_iter"], a["compactness"], a["min_size_factor"], a["subsample_stride"], a["convert_to_lab"])


def _run_cuda(img, K, a, rounds):
    from fast_slic_b200 import get_engine
    H, W, _ = img.shape
    eng = get_engine(H, W, K, 1, 0)
    t = torch.from_numpy(img).cuda()[None].contiguous()
    cl = eng.initialize_clusters(t)
    init = cl.cpu().numpy().copy()
    p = eng.params(*[a[k] for k in ("compactness", "min_size_factor", "subsample_stride", "convert_to_lab", "max_iter")])
    out = []
    for _ in range(rounds):
        lab = eng.iterate(t, cl, p, manhattan_spatial_dist=False)
        quad, pre = eng.debug_stages(1)
        out.append((lab[0].cpu().numpy().view(np.uint16), quad[0].cpu().numpy(), pre[0].cpu().numpy().view(np.uint16),
                    cl[0].cpu().numpy().copy()))
    return eng, init, out


def _compare_pipeline(euclid, name, img, K, a, rounds):
    eng, init, got = _run_cuda(img, K, a, rounds)
    cl = euclid.initialize(img, K)
    assert init.tobytes() == cl.tobytes(), name + ": initialize_clusters differs"
    for r, (glab, gquad, gpre, gcl) in enumerate(got):
        lab, quad, pre = euclid.iterate(img, cl, *_args(a), stages=True)
        assert (gquad == quad).all(), "%s round %d: quad image differs" % (name, r)
        assert (gpre == pre).all(), "%s round %d: pre-CCA labels differ (%d px)" % (name, r, int((gpre != pre).sum()))
        assert (glab == lab).all(), "%s round %d: final labels differ (%d px)" % (name, r, int((glab != lab).sum()))
        assert gcl.tobytes() == cl.tobytes(), "%s round %d: Cluster bytes differ" % (name, r)
    return eng


def _max_tile_candidates(clusters, S, W):
    """A lower bound on the longest candidate list of the assign kernels' warp tiles in the first pass: the clusters
    whose centre lies within S of a one-row, 32-column tile (a real tile has at least that many)."""
    cy, cx = clusters["y"].astype(int), clusters["x"].astype(int)
    best = 0
    for i in range(int(cy.max()) + 1):
        rows = np.abs(cy - i) <= S
        for j0 in range(0, W, 32):
            best = max(best, int((rows & (cx >= j0 - S) & (cx <= j0 + 31 + S)).sum()))
    return best


CASES = EUCLID_CASES + EUCLID_SAME_CASES


@pytest.mark.parametrize("group,case,seed", CASES, ids=[case_id(g, c) for g, c, _ in CASES])
def test_euclidean_pipeline(euclid, group, case, seed):
    """Slic(manhattan_spatial_dist=False) on the TMA kernel (its table), the LDG kernel, the generic kernel, the
    candidate-list overflow path of the warp tiles (assign_pixel_generic) and edge shapes and parameters."""
    name, kind, H, W, K, kw = case
    sigma, a = split_kwargs(kw)
    img = make_image(kind, H, W, seed=seed, sigma=sigma)
    eng = _compare_pipeline(euclid, name, img, K, a, 1)
    if group == "tma":
        assert eng.assign_impl() == 5, "the TMA-staged kernel did not run (impl %d)" % eng.assign_impl()
    elif group == "ldg":
        assert eng.assign_impl() == 4
    elif group == "generic":
        assert eng.S > 110 and eng.assign_impl() == 0
    elif group == "dense":
        assert eng.assign_impl() == 5
        assert _max_tile_candidates(euclid.initialize(img, K), eng.S, W) > AS_LIST, "no tile overflows its list"


def test_euclidean_warm_start(euclid):
    """A second iterate() on the clusters the first one left (the reference's video use)."""
    name, kind, H, W, K, kw = EUCLID_WARM_CASE
    sigma, a = split_kwargs(kw)
    _compare_pipeline(euclid, name, make_image(kind, H, W, seed=3, sigma=sigma), K, a, 2)


LDG_CASES = [c for c in EUCLID_CASES if c[0] in ("pipeline", "dense")]


@pytest.mark.parametrize("group,case,seed", LDG_CASES, ids=["%s-W%d" % (case_id(g, c), c[3] - 1) for g, c, _ in LDG_CASES])
def test_euclidean_ldg_kernel_by_width(euclid, group, case, seed):
    """The LDG kernel on these shapes one column narrower (W % 8 != 0 rules out the TMA kernel), its list overflow
    included (dense K)."""
    name, kind, H, W, K, kw = case
    W -= 1
    sigma, a = split_kwargs(kw)
    img = make_image(kind, H, W, seed=seed, sigma=sigma)
    eng = _compare_pipeline(euclid, name, img, K, a, 1)
    assert eng.assign_impl() == 4
    if group == "dense":
        assert _max_tile_candidates(euclid.initialize(img, K), eng.S, W) > AS_LIST, "no tile overflows its list"


VARIANTS = ("standard", "l2", "noq")
# the hand-picked cases under every variant, then the seeded sweep (variants 0 and 2 by seed)
REAL_PARAMS = [(v, c) for c in EUCLID_REAL_CASES for v in VARIANTS] + [(VARIANTS[v], c) for c, v in EUCLID_REAL_SWEEP]
REAL_IDS = ["%s_%dx%d_K%d-%s" % (c[:4] + (v,)) for c in EUCLID_REAL_CASES for v in VARIANTS] + \
           ["sweep%d_%s-%s" % (s, sweep_case_id(c), VARIANTS[v]) for s, (c, v) in enumerate(EUCLID_REAL_SWEEP)]


@pytest.mark.parametrize("variant,case", REAL_PARAMS, ids=REAL_IDS)
def test_euclidean_real_dist(euclid, variant, case):
    """SlicRealDist (coef * hypot, untruncated) and SlicRealDistNoQ (squared differences) with the flag off, cold and
    warm start: labels, pre-CCA labels, Cluster bytes and the variant's kernel; SlicRealDistL2 ignores the flag, as the
    reference does."""
    import fast_slic_b200 as fs
    kind, H, W, K, kw = case
    sigma, a = split_kwargs(kw)
    img = make_image(kind, H, W, seed=47, sigma=sigma)
    cls = {"standard": fs.SlicRealDist, "l2": fs.SlicRealDistL2, "noq": fs.SlicRealDistNoQ}[variant]
    make = lambda manhattan: cls(num_components=K, compactness=a["compactness"], min_size_factor=a["min_size_factor"],
                                 subsample_stride=a["subsample_stride"], convert_to_lab=a["convert_to_lab"],
                                 manhattan_spatial_dist=manhattan)
    s, plain = make(False), make(True)
    v = VARIANTS.index(variant)
    cl = euclid.initialize(img, K)
    for round_ in range(2):
        got = s.iterate(img, a["max_iter"]).view(np.uint16)
        want, want_pre = euclid.iterate_real(v, img, cl, *_args(a), stages=True)
        check_class_call("%s round %d" % (variant, round_), s, got, want, want_pre, cl, 10 + v, a["max_iter"])
        if v == 1:
            assert (plain.iterate(img, a["max_iter"]).view(np.uint16) == got).all()
            assert plain.slic_model.cluster_array.tobytes() == cl.tobytes()


PREEMPT_PARAMS = EUCLID_PREEMPT_CASES + EUCLID_PREEMPT_SWEEP
PREEMPT_IDS = [preempt_case_id(c) for c in EUCLID_PREEMPT_CASES] + \
              ["%s_%s_t%g" % (preempt_sweep_id(s), sweep_case_id(c), c[4]) for s, c in enumerate(EUCLID_PREEMPT_SWEEP)]


@pytest.mark.parametrize("case", PREEMPT_PARAMS, ids=PREEMPT_IDS)
def test_euclidean_preemptive(euclid, case):
    """Slic(preemptive=True, manhattan_spatial_dist=False), cold and warm start: labels, pre-CCA labels, Cluster bytes
    and k_assign_preempt on the update passes."""
    import fast_slic_b200 as fs
    kind, H, W, K, thres, kw = case
    sigma, a = split_kwargs(kw)
    img = make_image(kind, H, W, seed=53, sigma=sigma)
    s = fs.Slic(num_components=K, compactness=a["compactness"], min_size_factor=a["min_size_factor"],
                subsample_stride=a["subsample_stride"], convert_to_lab=a["convert_to_lab"], preemptive=True,
                preemptive_thres=thres, manhattan_spatial_dist=False)
    cl = euclid.initialize(img, K)
    for round_ in range(2):
        got = s.iterate(img, a["max_iter"]).view(np.uint16)
        want, _, want_pre = euclid.iterate(img, cl, *_args(a), stages=True, preemptive=True, preemptive_thres=thres)
        check_class_call("round %d" % round_, s, got, want, want_pre, cl, PREEMPT, a["max_iter"])


def test_euclidean_iterate_batch(euclid):
    """iterate_batch() with host and device batches, for Slic, the float-distance classes and preemptive."""
    import fast_slic_b200 as fs
    H, W, K, B = 120, 160, 48, 3
    imgs = np.stack([make_image("syn" if b != 1 else "blocks", H, W, seed=810 + b) for b in range(B)])
    for name, obj, ref_call in (
            ("slic", fs.Slic(num_components=K, manhattan_spatial_dist=False),
             lambda im, cl: euclid.iterate(im, cl)),
            ("standard", fs.SlicRealDist(num_components=K, manhattan_spatial_dist=False),
             lambda im, cl: euclid.iterate_real(0, im, cl)),
            ("noq", fs.SlicRealDistNoQ(num_components=K, manhattan_spatial_dist=False),
             lambda im, cl: euclid.iterate_real(2, im, cl)),
            ("preemptive", fs.Slic(num_components=K, preemptive=True, preemptive_thres=0.1, manhattan_spatial_dist=False),
             lambda im, cl: euclid.iterate(im, cl, preemptive=True, preemptive_thres=0.1))):
        lab_h, cl_h = obj.iterate_batch(imgs, return_clusters=True)
        lab_d, cl_d = obj.iterate_batch(torch.from_numpy(imgs).cuda(), return_clusters=True)
        for b in range(B):
            cl = euclid.initialize(imgs[b], K)
            want = ref_call(imgs[b], cl)
            assert (lab_h[b].view(np.uint16) == want).all(), (name, "host", b)
            assert cl_h[b].tobytes() == cl.tobytes(), (name, "host clusters", b)
            assert (lab_d[b].cpu().numpy().view(np.uint16) == want).all(), (name, "device", b)
            assert cl_d[b].cpu().numpy().tobytes() == cl.tobytes(), (name, "device clusters", b)


def test_euclidean_stream(euclid):
    """SlicStream(manhattan_spatial_dist=False), cold start per batch and warm start across batches."""
    from fast_slic_b200 import SlicStream
    H, W, K, B, T = 120, 160, 40, 3, 3
    frames = [np.stack([make_image("syn", H, W, seed=900 + 10 * b + t, sigma=10.0 + t) for b in range(B)]) for t in range(T)]
    for warm in (False, True):
        st = SlicStream(H, W, K, batch=B, depth=2, min_size_factor=0.1, warm_start=warm, manhattan_spatial_dist=False)
        got = list(st.map(frames))
        st.close()
        for b in range(B):
            cl = euclid.initialize(frames[0][b], K)
            for t in range(T):
                if not warm:
                    cl = euclid.initialize(frames[t][b], K)
                want = euclid.iterate(frames[t][b], cl, 10, 10.0, 0.1, 3, True)
                assert (got[t][b].view(np.uint16) == want).all(), (warm, b, t)


# Manhattan (True) / Euclidean (False) on one context.  Calls 2, 6 and 8 capture a graph (the same key came twice),
# call 4 replays the Manhattan graph between two plain Euclidean calls: the plain call after it must not reuse the
# spatial patches the replay left.
CACHE_SEQUENCE = [True, True, False, True, False, False, True, True, False, True]


def test_euclidean_cache_alternation(euclid):
    """One cached context alternating the flag on the graph-replay path (device API, 2 images, same buffers,
    non-default stream) and on the host path: every call against the checker, clusters carried over."""
    from fast_slic_b200 import Engine
    H, W, K, B = 120, 160, 40, 2
    imgs = np.stack([make_image("syn", H, W, seed=950 + b) for b in range(B)])
    eng = Engine(H, W, K, B)
    p = eng.params(10.0, 0.1, 3, True, 10)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        d_img = torch.from_numpy(imgs).cuda()
        cl = eng.initialize_clusters(d_img)
        lab = torch.empty((B, H, W), dtype=torch.int16, device="cuda")
        dev = []
        for m in CACHE_SEQUENCE:
            eng.iterate(d_img, cl, p, lab, manhattan_spatial_dist=m)
            dev.append((lab.clone(), cl.clone()))
    st.synchronize()
    cl_h = eng.initialize_clusters_host(imgs)
    host = []
    for m in CACHE_SEQUENCE:
        labels = eng.iterate_host(imgs, cl_h, p, manhattan_spatial_dist=m)
        host.append((labels.copy(), cl_h.copy()))
    eng.close()
    for b in range(B):
        c_dev, c_host = euclid.initialize(imgs[b], K), euclid.initialize(imgs[b], K)
        for t, m in enumerate(CACHE_SEQUENCE):
            want = euclid.iterate(imgs[b], c_dev, 10, 10.0, 0.1, 3, True, manhattan=m)
            assert (dev[t][0][b].cpu().numpy().view(np.uint16) == want).all(), ("device", b, t, m)
            assert dev[t][1][b].cpu().numpy().tobytes() == c_dev.tobytes(), ("device clusters", b, t, m)
            want = euclid.iterate(imgs[b], c_host, 10, 10.0, 0.1, 3, True, manhattan=m)
            assert (host[t][0][b].view(np.uint16) == want).all(), ("host", b, t, m)
            assert host[t][1][b].tobytes() == c_host.tobytes(), ("host clusters", b, t, m)
