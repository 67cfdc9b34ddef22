"""The default integer path (Slic, with the Manhattan and the Euclidean spatial term) on the GPU over its seeded sweep
and the two ends of the compactness range, against the checker (the compiled reference where it was built, else the
restatement tests/test_default_sweep_cpu.py pins to the reference's digests).  Tolerance 0: labels, pre-CCA labels,
the Lab quad image and raw Cluster bytes, cold start and warm start.

Every call goes through each entry point that takes a different route through the library: Slic.iterate (the host
path), Engine.iterate (the device path), iterate_batch on a numpy array (host batches: graph replay below 4 images,
two overlapping lanes from 16) and on a cuda tensor (TPS = 4 super tiles and the non-fused prepare kernels)."""
import numpy as np
import pytest
import torch

from cases import SWEEP_KINDS, make_image, split_kwargs, sweep_S
from default_sweep_cases import LIMIT_SHAPES, all_cases, case_key, compactness_limit, next_float_up

pytestmark = pytest.mark.gpu

# what the calls of this file reached: ("update" | "full", kernel, tps), ("prepare", code), ("fused",)
REACHED = set()


def _record(eng):
    d = eng.dispatch()
    for p in ("update", "full"):
        if d[p]["kernel"] >= 0:
            REACHED.add((p, d[p]["kernel"], d[p]["tps"]))
    if d["prepare"]:
        REACHED.add(("prepare", d["prepare"]))
    if d["fused_prepares"] > 0:
        REACHED.add(("fused",))
    return d


class Checkers:
    """family 0: the session checker (Manhattan); family 1: the Euclidean one, chosen as test_euclidean_gpu.py does."""

    def __init__(self, checker):
        from oracle_euclid.euclid import Port, Ref
        self.c = checker
        self.kind = checker.kind
        self.euclid = Ref() if Ref.available() else Port()
        self.ekw = dict(arch="x64/avx2", num_threads=checker._threads) if Ref.available() else {}

    def initialize(self, img, K):
        return self.c.initialize(img, K)

    def iterate(self, family, img, cl, a):
        args = (a["max_iter"], a["compactness"], a["min_size_factor"], a["subsample_stride"], a["convert_to_lab"])
        if family == 0:
            return self.c.iterate(img, cl, *args, stages=True)
        return self.euclid.iterate(img, cl, *args, stages=True, **self.ekw)

    def rounds(self, family, img, K, a, n=2):
        """(initial Cluster bytes, [(labels, quad, pre-CCA labels, Cluster bytes)] of n calls on carried clusters)."""
        cl = self.initialize(img, K)
        init = cl.tobytes()
        out = []
        for _ in range(n):
            lab, quad, pre = self.iterate(family, img, cl, a)
            out.append((lab, quad, pre, cl.tobytes()))
        return init, out


@pytest.fixture(scope="module")
def checkers(checker):
    return Checkers(checker)


def _slic(K, a, family, **kw):
    from fast_slic_b200 import Slic
    return Slic(num_components=K, compactness=a["compactness"], min_size_factor=a["min_size_factor"],
                subsample_stride=a["subsample_stride"], convert_to_lab=a["convert_to_lab"],
                manhattan_spatial_dist=family == 0, **kw)


def _params(a):
    from fast_slic_b200 import Engine
    return Engine.params(a["compactness"], a["min_size_factor"], a["subsample_stride"], a["convert_to_lab"], a["max_iter"])


def _np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else t


def _compare(name, want, lab=None, quad=None, pre=None, cl=None):
    wlab, wquad, wpre, wcl = want
    if quad is not None:
        quad = _np(quad)
        assert (quad == wquad).all(), "%s: quad image differs (%d px)" % (name, int((quad != wquad).any(-1).sum()))
    if pre is not None:
        pre = _np(pre).view(np.uint16)
        assert (pre == wpre).all(), "%s: pre-CCA labels differ (%d px)" % (name, int((pre != wpre).sum()))
    if lab is not None:
        lab = _np(lab).view(np.uint16)
        assert (lab == wlab).all(), "%s: labels differ (%d px)" % (name, int((lab != wlab).sum()))
    if cl is not None:
        assert np.ascontiguousarray(_np(cl)).tobytes() == wcl, "%s: Cluster bytes differ" % name


def _image(case, seed, kind=None):
    _, k, H, W, _, kw = case
    sigma, _ = split_kwargs(kw)
    return make_image(kind or k, H, W, seed=seed, sigma=sigma)


PARAMS = [(f, g, c, s) for f in (0, 1) for g, c, s in all_cases(f)]
IDS = [case_key(f, g, c) for f, g, c, _ in PARAMS]


@pytest.mark.parametrize("family,group,case,seed", PARAMS, ids=IDS)
def test_single_image(checkers, family, group, case, seed):
    """One image through Engine.iterate (device buffers) and through Slic.iterate (the host entry point), cold then warm
    on the clusters the first call left."""
    from fast_slic_b200 import get_engine
    _, _, H, W, K, kw = case
    _, a = split_kwargs(kw)
    img = _image(case, seed)
    init, want = checkers.rounds(family, img, K, a)
    eng = get_engine(H, W, K, 1)
    t = torch.from_numpy(img).cuda()[None].contiguous()
    cl = eng.initialize_clusters(t)
    assert cl[0].cpu().numpy().tobytes() == init, "initialize_clusters differs"
    for r in range(2):
        lab = eng.iterate(t, cl, _params(a), manhattan_spatial_dist=family == 0)
        _record(eng)
        quad, pre = eng.debug_stages(1)
        _compare("device round %d" % r, want[r], lab[0], quad[0], pre[0], cl[0])
    if group == "limit" and a["compactness"] > 0:  # one float more is refused, and the call writes nothing
        from fast_slic_b200._lib import FslicError
        before = (lab.clone(), cl.clone())
        with pytest.raises(FslicError, match="compactness too large"):
            eng.iterate(t, cl, _params(dict(a, compactness=next_float_up(a["compactness"]))), lab,
                        manhattan_spatial_dist=family == 0)
        assert torch.equal(lab, before[0]) and torch.equal(cl, before[1]), "a refused call wrote"
    s = _slic(K, a, family)
    for r in range(2):
        lab = s.iterate(img, a["max_iter"])
        eng = get_engine(H, W, K, 1)
        _record(eng)
        quad, pre = eng.debug_stages(1)
        _compare("host round %d" % r, want[r], lab, quad[0], pre[0], s.slic_model.cluster_array)


def _three_kinds(kind):
    return (kind,) + tuple(k for k in SWEEP_KINDS if k != kind)[:2]


def _check_batch(checkers, family, case, imgs, where, rounds=2, stages=True, expect=None):
    """iterate_batch of `imgs` (numpy, or a cuda tensor with where == "device"): every image against its single-image
    checker result, cold and then warm on the clusters the batch returned.  `expect`: dispatch fields the last call
    must show ({"update_tps": 4, "prepare": 1, ...})."""
    from fast_slic_b200 import get_engine
    _, _, H, W, K, kw = case
    _, a = split_kwargs(kw)
    B = imgs.shape[0]
    want = [checkers.rounds(family, imgs[b], K, a, rounds) for b in range(B)]
    s = _slic(K, a, family)
    src = torch.from_numpy(imgs).cuda() if where == "device" else imgs
    cl = None
    for r in range(rounds):
        lab, cl = s.iterate_batch(src, max_iter=a["max_iter"], clusters=cl, return_clusters=True)
        eng = get_engine(H, W, K, B)
        d = _record(eng)
        quad, pre = eng.debug_stages(B) if stages else (None, None)
        for b in range(B):
            _compare("%s batch of %d, image %d, round %d" % (where, B, b, r), want[b][1][r], lab[b],
                     None if quad is None else quad[b], None if pre is None else pre[b], cl[b])
        for k, v in (expect or {}).items():
            got = d["update"]["tps"] if k == "update_tps" else d[k]
            assert got == v, "%s batch of %d: dispatch %s = %r, expected %r" % (where, B, k, got, v)
    return want


@pytest.mark.parametrize("family,group,case,seed", PARAMS, ids=IDS)
def test_batch_of_three(checkers, family, group, case, seed):
    """Three images of different kinds through iterate_batch, on a numpy array (host pipeline, CUDA graph captured on
    the first call and replayed on the second) and on a cuda tensor; each image equals its single-image result."""
    _, kind, H, W, K, kw = case
    imgs = np.stack([_image(case, seed + 7 * b, k) for b, k in enumerate(_three_kinds(kind))])
    for where in ("host", "device"):
        _check_batch(checkers, family, case, imgs, where)


# ---- large batches at the edges --------------------------------------------------------------------------------------
def _hd_case(at_limit):
    """720p, K = 1600 (S = 24), the TMA kernel's shape of bench.py, at an end of the compactness range."""
    c = compactness_limit(24, True) if at_limit else 0.0
    return ("hd_%s" % ("limit" if at_limit else "c0"), "syn", 720, 1280, 1600,
            dict(compactness=c, min_size_factor=0.0, max_iter=4))


def _hd_images(n, seed):
    kinds = ("syn", "syn", "blocks", "noise")
    return np.stack([make_image(kinds[b % 4], 720, 1280, seed=seed + b, sigma=(12.0, 40.0)[b % 2]) for b in range(n)])


@pytest.mark.parametrize("family", [0, 1], ids=["manhattan", "euclid"])
@pytest.mark.parametrize("at_limit", [True, False], ids=["limit", "c0"])
def test_hd_batch_of_17(checkers, family, at_limit):
    """17 images at 720p: the host call splits into two overlapping lanes of 8 and 9 images, the device call is one
    launch of 17 whose update passes take super tiles of 4 warp tiles (TPS = 4: 600 super tiles per image, 10200 >=
    132 SMs x 32 warps)."""
    case = _hd_case(at_limit)
    imgs = _hd_images(17, 300 + 40 * family + 20 * at_limit)
    _check_batch(checkers, family, case, imgs, "device", rounds=1, expect={"update_tps": 4})
    _check_batch(checkers, family, case, imgs, "host", rounds=1)


def _bigk_case():
    """K > 4096 (S = 3) at the compactness limit: the prepare kernels of large K."""
    return ("bigK_240x320_K5000_limit", "syn", 240, 320, 5000,
            dict(compactness=compactness_limit(3, True), min_size_factor=0.0, max_iter=5))


@pytest.mark.parametrize("B,prepare", [(8, 1), (3, 2)], ids=["B8_k_prepare", "B3_k_prepare2"])
def test_large_K_batches(checkers, B, prepare):
    """K > 4096: k_prepare from 8 images up, k_prepare2 below (device calls); the host calls take the split-upload
    pipeline (8 images) and the graph replay (3)."""
    case = _bigk_case()
    imgs = np.stack([make_image(SWEEP_KINDS[b % 3], 240, 320, seed=400 + b) for b in range(B)])
    _check_batch(checkers, 0, case, imgs, "device", expect={"prepare": prepare})
    _check_batch(checkers, 0, case, imgs, "host")


SUB_BATCH_CASES = [(f, g, c, s) for f, g, c, s in PARAMS if g == "limit" and c[0].startswith(("S2_", "S20_syn", "S125_"))
                   and c[-1]["convert_to_lab"] == (f == 0)]


@pytest.mark.parametrize("family,group,case,seed", SUB_BATCH_CASES, ids=[case_key(f, g, c) for f, g, c, _ in SUB_BATCH_CASES])
def test_sub_batched_edges(checkers, monkeypatch, family, group, case, seed):
    """Connectivity enforcement in sub-batches of 2 and the host pipeline in chunks of 3, on 7 images at the ends of the
    compactness range: labels and Cluster bytes (the pre-CCA stage of a chunked host call holds its last chunk only)."""
    from fast_slic_b200 import clear_engine_cache
    monkeypatch.setenv("FSLIC_CCA_BATCH", "2")
    monkeypatch.setenv("FSLIC_HOST_CHUNK", "3")
    clear_engine_cache()
    try:
        imgs = np.stack([_image(case, seed + 11 * b, SWEEP_KINDS[b % 4]) for b in range(7)])
        _check_batch(checkers, family, case, imgs, "host", rounds=1, stages=False)
        _check_batch(checkers, family, case, imgs, "device", rounds=1)
    finally:
        clear_engine_cache()


# ---- the spatial patch cache -----------------------------------------------------------------------------------------
def test_patch_cache_across_compactness(checkers):
    """k_build_sptable's patches are kept across calls with equal (S, stride, coef, distance).  One context alternates
    compactness limit -> 0 -> 10 -> limit with Lab on and off and both distances, on device buffers (2 images) and on
    the host path (graph captured and replayed): every call equals the checker, clusters carried over."""
    from fast_slic_b200 import Engine
    H, W, K, B = 200, 264, 130, 2
    S = sweep_S(H, W, K)
    imgs = np.stack([make_image(k, H, W, seed=500 + b) for b, k in enumerate(("syn", "blocks"))])
    seq = [(family, lab, c) for lab in (True, False) for family in (0, 1)
           for c in (compactness_limit(S, lab), 0.0, 10.0, compactness_limit(S, lab))]
    eng = Engine(H, W, K, B)
    try:
        d_img = torch.from_numpy(imgs).cuda()
        d_cl = eng.initialize_clusters(d_img)
        lab_d = torch.empty((B, H, W), dtype=torch.int16, device="cuda")
        h_cl = eng.initialize_clusters_host(imgs)
        want_cl = [checkers.initialize(imgs[b], K) for b in range(B)]
        host_cl = [c.copy() for c in want_cl]
        for t, (family, lab, c) in enumerate(seq):
            a = dict(max_iter=5, compactness=c, min_size_factor=0.1, subsample_stride=3, convert_to_lab=lab)
            p = _params(a)
            eng.iterate(d_img, d_cl, p, lab_d, manhattan_spatial_dist=family == 0)
            _record(eng)
            quad, pre = eng.debug_stages(B)
            for b in range(B):
                wl, wq, wp = checkers.iterate(family, imgs[b], want_cl[b], a)
                _compare("device call %d %r image %d" % (t, (family, lab, c), b), (wl, wq, wp, want_cl[b].tobytes()),
                         lab_d[b], quad[b], pre[b], d_cl[b])
            h_lab = eng.iterate_host(imgs, h_cl, p, manhattan_spatial_dist=family == 0)
            _record(eng)
            for b in range(B):
                wl, wq, wp = checkers.iterate(family, imgs[b], host_cl[b], a)
                _compare("host call %d %r image %d" % (t, (family, lab, c), b), (wl, wq, wp, host_cl[b].tobytes()),
                         h_lab[b], None, None, h_cl[b])
    finally:
        eng.close()


# ---- the refusal above the limit ------------------------------------------------------------------------------------
REFUSAL_SHAPES = [s for s in LIMIT_SHAPES if s[0].startswith(("S1_", "S20_syn", "S125_"))]
SENTINEL = 0x5A5A


@pytest.mark.parametrize("family", [0, 1], ids=["manhattan", "euclid"])
@pytest.mark.parametrize("lab", [True, False], ids=["lab", "rgb"])
@pytest.mark.parametrize("shape", REFUSAL_SHAPES, ids=[s[0] for s in REFUSAL_SHAPES])
def test_refuses_the_next_float_above_the_limit(checkers, shape, lab, family):
    """compactness = the next float32 above the limit raises FslicError "compactness too large" from Slic.iterate,
    iterate_batch (numpy and tensor), Engine.iterate, Engine.iterate_host and Engine.iterate_preemptive, and writes
    nothing: label and cluster buffers come back as they went in.  The next accepted call on the same context (the
    limit itself) equals the checker."""
    from fast_slic_b200 import get_engine
    from fast_slic_b200._lib import FslicError
    name, kind, H, W, K, kw = shape
    limit = compactness_limit(sweep_S(H, W, K), lab)
    bad = next_float_up(limit)
    _, a_ok = split_kwargs(dict(kw, compactness=limit, convert_to_lab=lab))
    a_bad = dict(a_ok, compactness=bad)
    manhattan = family == 0
    img = make_image(kind, H, W, seed=77)
    init, want = checkers.rounds(family, img, K, a_ok, 1)
    refused = dict(match="compactness too large")

    s = _slic(K, a_bad, family)
    with pytest.raises(FslicError, **refused):
        s.iterate(img, a_bad["max_iter"])
    assert s.slic_model.cluster_array.tobytes() == init, "Slic.iterate: clusters changed by a refused call"
    s.compactness = limit
    _compare("Slic.iterate after the refusal", want[0], s.iterate(img, a_ok["max_iter"]), cl=s.slic_model.cluster_array)

    imgs = np.stack([img, img])
    with pytest.raises(FslicError, **refused):
        _slic(K, a_bad, family).iterate_batch(imgs, max_iter=a_bad["max_iter"])
    with pytest.raises(FslicError, **refused):
        _slic(K, a_bad, family).iterate_batch(torch.from_numpy(imgs).cuda(), max_iter=a_bad["max_iter"])

    eng = get_engine(H, W, K, 2)
    h_cl = eng.initialize_clusters_host(imgs)
    h_cl0 = h_cl.copy()
    h_lab = np.full((2, H, W), SENTINEL, np.uint16).view(np.int16)
    with pytest.raises(FslicError, **refused):
        eng.iterate_host(imgs, h_cl, _params(a_bad), h_lab, manhattan_spatial_dist=manhattan)
    assert h_cl.tobytes() == h_cl0.tobytes() and (h_lab.view(np.uint16) == SENTINEL).all(), "iterate_host wrote"
    eng.iterate_host(imgs, h_cl, _params(a_ok), h_lab, manhattan_spatial_dist=manhattan)
    for b in range(2):
        _compare("iterate_host after the refusal, image %d" % b, want[0], h_lab[b], cl=h_cl[b])

    d_img = torch.from_numpy(imgs).cuda()
    d_cl = eng.initialize_clusters(d_img)
    d_cl0 = d_cl.clone()
    d_lab = torch.full((2, H, W), SENTINEL, dtype=torch.int16, device="cuda")
    d_lab0 = d_lab.clone()
    for call in (lambda p: eng.iterate(d_img, d_cl, p, d_lab, manhattan_spatial_dist=manhattan),
                 lambda p: eng.iterate_preemptive(d_img, d_cl, p, 0.05, d_lab, manhattan_spatial_dist=manhattan)):
        with pytest.raises(FslicError, **refused):
            call(_params(a_bad))
        assert torch.equal(d_cl, d_cl0) and torch.equal(d_lab, d_lab0), "a refused device call wrote"
    eng.iterate(d_img, d_cl, _params(a_ok), d_lab, manhattan_spatial_dist=manhattan)
    quad, pre = eng.debug_stages(2)
    for b in range(2):
        _compare("Engine.iterate after the refusal, image %d" % b, want[0], d_lab[b], quad[b], pre[b], d_cl[b])


# ---- what the file reached --------------------------------------------------------------------------------------------
NEEDED = {("update", 5, 1): "TMA kernel update pass with tps 1", ("update", 5, 4): "TMA kernel update pass with tps 4",
          ("update", 4): "LDG kernel update pass", ("update", 0): "generic kernel update pass",
          ("prepare", 1): "k_prepare", ("prepare", 2): "k_prepare2", ("prepare", 3): "k_prepare3",
          ("fused",): "a prepare fused into the TMA kernel's tail"}


def _reached(key):
    if key[0] == "update" and len(key) == 2:
        return any(r[:2] == key for r in REACHED)
    return key in REACHED


def test_dispatch_coverage(request):
    """The calls above reached every update-pass kernel (TMA with 1 and with 4 warp tiles per super tile, LDG,
    generic), every prepare kernel and the fused prepare.  Runs last; skipped when tests of this file were deselected."""
    mine = [i for i in request.session.items if i.module is request.module and i.name != request.node.name]
    from_file = [n for n in dir(request.module) if n.startswith("test_") and n != "test_dispatch_coverage"]
    if {i.originalname for i in mine} != set(from_file) or len(REACHED) == 0:
        pytest.skip("only part of the file ran")
    print("dispatch reached:", sorted(REACHED))
    missed = [what for key, what in NEEDED.items() if not _reached(key)]
    assert not missed, "never reached: " + ", ".join(missed)
