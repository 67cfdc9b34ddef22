"""Launch branches that only large batches and large images reach, against the CPU checkers at tolerance 0.

Every case runs a batch of different images (image kinds mixed across the slots, so that a slot-indexing mistake shows
up), a cold call and then a warm call on the clusters the first one left, and compares each image with its own
single-image checker run: labels, pre-CCA labels and raw Cluster bytes.  The checker result of an image and round is
computed once and compared with the device-entry and the host-entry outputs.  Every case also reads back the launch
decisions of its calls (Engine.dispatch()) and asserts the branch it is there for: if a heuristic change moves a shape
off its branch, the test fails and says so instead of quietly testing something else.
"""
import numpy as np
import pytest
import torch

from cases import make_image

pytestmark = pytest.mark.gpu

KINDS = ("syn", "noise", "blocks", "tiled")
TMA, LDG, GENERIC, PREEMPT, LSC = 5, 4, 0, 13, 14
REAL = {"standard": 10, "l2": 11, "noq": 12}
K_PREPARE3, K_PREPARE2, K_PREPARE = 3, 2, 1


def _cdiv(a, b):
    return -(-a // b)


def _batch(H, W, B, seed):
    """B different images; slot b gets kind KINDS[b % 4]."""
    return np.stack([make_image(KINDS[b % len(KINDS)], H, W, seed=seed + b) for b in range(B)])


# ---- checkers: fn(image, clusters) -> (labels, pre-CCA labels), clusters updated in place ----------------------------
def _slic(impl, msf, **kw):
    def run(img, cl):
        res = impl.iterate(img, cl, 10, 10.0, msf, 3, True, stages=True, **kw)
        return res[0], res[-1]
    return run


def _real(impl, v, msf):
    def run(img, cl):
        res = impl.iterate_real(v, img, cl, 10, 10.0, msf, 3, True, stages=True)
        return res[0], res[-1]
    return run


def _lsc(impl, msf):
    def run(img, cl):
        lab, st = impl.iterate_lsc(img, cl, 10, 10.0, msf, 3, True, stages=True)
        return lab, st["pre"]
    return run


class _Euclid:
    """The Euclidean checker (manhattan_spatial_dist=False), chosen as test_euclidean_gpu.py chooses it."""

    def __init__(self, checker):
        from oracle_euclid.euclid import Port, Ref
        self.reference = Ref.available()
        self._impl = Ref() if self.reference else Port()
        self._kw = dict(arch="x64/avx2", num_threads=checker._threads) if self.reference else {}

    def iterate(self, img, cl, *a, **kw):
        return self._impl.iterate(img, cl, *a, **kw, **self._kw)

    def iterate_real(self, v, img, cl, *a, **kw):
        return self._impl.iterate_real(v, img, cl, *a, **kw)


@pytest.fixture(scope="module")
def euclid(checker):
    return _Euclid(checker)


@pytest.fixture(scope="module")
def lsc_checker():
    from oracle_lsc.lsc import Port, Ref
    return Ref() if Ref.available() else Port()


def _want(checker, fn, imgs, K):
    """Per image: [(labels, pre-CCA labels, Cluster bytes) of the cold round, ... of the warm round]."""
    out = []
    for img in imgs:
        cl = checker.initialize(img, K)
        rounds = []
        for _ in range(2):
            lab, pre = fn(img, cl)
            rounds.append((lab, pre, cl.tobytes()))
        out.append(rounds)
    return out


def _compare(name, got, want):
    """got: [(labels [B,H,W] u16, pre-CCA labels [B,H,W] u16, clusters [B] (raw records per image)) per round]."""
    for r, (lab, pre, cl) in enumerate(got):
        assert len(lab) == len(want), name
        for b, w in enumerate(want):
            wlab, wpre, wcl = w[r]
            where = "%s round %d image %d" % (name, r, b)
            assert (pre[b] == wpre).all(), "%s: pre-CCA labels differ (%d px)" % (where, int((pre[b] != wpre).sum()))
            assert (lab[b] == wlab).all(), "%s: labels differ (%d px)" % (where, int((lab[b] != wlab).sum()))
            assert cl[b].tobytes() == wcl, "%s: Cluster bytes differ" % where


# ---- runs: [(labels, pre, clusters, dispatch) per round] ----------------------------------------------------------------
def _pre(eng, B):
    return eng.debug_stages(B)[1].cpu().numpy().view(np.uint16)


def _device(eng, imgs, p, manhattan=True):
    t = torch.from_numpy(imgs).cuda()
    cl = eng.initialize_clusters(t)
    out = []
    for _ in range(2):
        lab = eng.iterate(t, cl, p, manhattan_spatial_dist=manhattan)
        out.append((lab.cpu().numpy().view(np.uint16), _pre(eng, len(imgs)), cl.cpu().numpy(), eng.dispatch()))
    return out


def _host(eng, imgs, p, manhattan=True):
    cl = eng.initialize_clusters_host(imgs)
    out = []
    for _ in range(2):
        lab = eng.iterate_host(imgs, cl, p, manhattan_spatial_dist=manhattan)
        out.append((lab.view(np.uint16), _pre(eng, len(imgs)), cl.copy(), eng.dispatch()))
    return out


def _check(name, runs, want, expect):
    """Outputs of every round against the checker, then `expect(name, dispatch)` on the read-back of every round."""
    _compare(name, [r[:3] for r in runs], want)
    for r, run in enumerate(runs):
        expect("%s round %d" % (name, r), run[3])


def _assert_pass(name, d, which, kernel, items, tps=1, min_trips=2):
    """The `which` pass ("update": the last update pass, "full") of read-back d ran `kernel` over `items` work items
    (super tiles of `tps` tiles, or pixels) in at least `min_trips` rounds of its grid-stride walk."""
    p = d[which]
    msg = "%s: the %s pass left its branch (kernel %s, tps %d, %d trips expected; read back %r)" % (
        name, which, kernel, tps, min_trips, d)
    assert p["kernel"] == kernel and p["tps"] == tps and p["items"] == items, msg
    assert p["trips"] == _cdiv(p["items"], p["grid"] * p["workers"]), msg
    assert p["trips"] >= min_trips, msg


def _tiles(H, W, B, tps, stride, rem):
    """Super tiles of one pass of the tile kernels: rows rem, rem + stride, ... in warp tiles of 4 sub-rows x 32."""
    return _cdiv(_cdiv(W, 32), tps) * _cdiv(_cdiv(H - rem, stride), 4) * B


def _pixels(H, W, B, stride, rem):
    return _cdiv(H - rem, stride) * W * B


def _assert_walk_carries(name, d, which, W, B):
    """The tile kernels walk their super tiles (b, ty, sx) by a fixed step of grid x warps super tiles, with a carry from
    sx into ty and from ty into b instead of a division.  When the step is a whole number of super-tile rows (or of
    images) some of those carries never run, and the walk is not tested.  The step is a run-time value (SM count,
    occupancy, warps per CTA): check the read-back, so that a GPU or heuristic on which the shape stops exercising the
    carries fails here instead of passing without testing them."""
    p = d[which]
    stx = _cdiv(_cdiv(W, 32), p["tps"])
    per_img = p["items"] // B
    rest = (p["grid"] * p["workers"]) % per_img
    assert rest % stx != 0, "%s: the %s pass's walk step is a whole number of super-tile rows (%d super tiles per row, " \
        "%d per image): its carries do not run; read back %r" % (name, which, stx, per_img, d)


LAST_REM = (10 - 1) % 3  # sub-row offset of the last of the 10 update passes at stride 3


# ---- 1. LDG warp-tile kernel with 4-tile super tiles (W % 8 != 0) --------------------------------------------------------
# 768 x 1246: W % 8 = 6 (LDG kernel), 39 warp tiles per row, so 10 super tiles per row, the last one holding 3 tiles.  (At
# 768 x 1366 the rows have 11 super tiles, and on a 132-SM H100 the walk step, 264 CTAs x 16 warps, is a multiple of 11 and
# of a whole image: no carry runs.)
LDG_SHAPE = (768, 1246, 1600)


def _expect_ldg(H, W, B, upd_tps):
    def check(name, d):
        _assert_pass(name, d, "update", LDG, _tiles(H, W, B, upd_tps, 3, LAST_REM), upd_tps, 2 if upd_tps == 4 else 1)
        _assert_pass(name, d, "full", LDG, _tiles(H, W, B, 4, 1, 0), 4)
        _assert_walk_carries(name, d, "update", W, B)
        _assert_walk_carries(name, d, "full", W, B)
    return check


def test_ldg_super_tiles(checker):
    """k_assign_warp on super tiles of 4 tiles, several per warp, walking across image boundaries.  B = 16 through the
    device entry and through the host entry (two half pipelines of 8); then B = 4 on the same context, where the update
    passes get single tiles and the full pass super tiles."""
    from fast_slic_b200 import Engine
    H, W, K = LDG_SHAPE
    B = 16
    assert W % 8 != 0
    imgs = _batch(H, W, B, seed=1000)
    want = _want(checker, _slic(checker, 0.1), imgs, K)
    eng = Engine(H, W, K, B)
    try:
        p = eng.params(10.0, 0.1, 3, True, 10)
        _check("device B=16", _device(eng, imgs, p), want, _expect_ldg(H, W, 16, 4))
        _check("host B=16", _host(eng, imgs, p), want, _expect_ldg(H, W, 8, 4))
        _check("device B=4", _device(eng, imgs[:4], p), want[:4], _expect_ldg(H, W, 4, 1))
    finally:
        eng.close()


def test_ldg_super_tiles_euclidean(euclid, checker):
    """The same LDG super-tile walk with manhattan_spatial_dist=False, against the Euclidean checker."""
    from fast_slic_b200 import Engine
    H, W, K = LDG_SHAPE
    B = 16
    imgs = _batch(H, W, B, seed=1100)
    want = _want(checker, _slic(euclid, 0.1), imgs, K)
    eng = Engine(H, W, K, B)
    try:
        p = eng.params(10.0, 0.1, 3, True, 10)
        _check("euclidean device B=16", _device(eng, imgs, p, manhattan=False), want, _expect_ldg(H, W, B, 4))
    finally:
        eng.close()


# ---- 2. TMA kernel with a ragged last super tile --------------------------------------------------------------------------
def test_tma_ragged_super_tiles(checker):
    """768 x 1248: W % 8 == 0 (TMA kernel) but 39 warp tiles per row, so the last super tile of every row holds 3 tiles
    (and, as for the LDG shape, 10 super tiles per row keep the walk's carries running).  B = 16 through the device entry
    and the host entry (two halves of 8)."""
    from fast_slic_b200 import Engine
    H, W, K, B = 768, 1248, 1600, 16
    assert W % 8 == 0 and _cdiv(W, 32) % 4 != 0
    imgs = _batch(H, W, B, seed=1200)
    want = _want(checker, _slic(checker, 0.1), imgs, K)

    def expect(B_slice):
        def check(name, d):
            _assert_pass(name, d, "update", TMA, _tiles(H, W, B_slice, 4, 3, LAST_REM), 4)
            _assert_walk_carries(name, d, "update", W, B_slice)
            assert d["full"]["kernel"] == TMA, "%s: the full pass left the TMA kernel: %r" % (name, d)
        return check

    eng = Engine(H, W, K, B)
    try:
        p = eng.params(10.0, 0.1, 3, True, 10)
        _check("device B=16", _device(eng, imgs, p), want, expect(16))
        _check("host B=16", _host(eng, imgs, p), want, expect(8))
    finally:
        eng.close()


# ---- 3. prepare kernels ---------------------------------------------------------------------------------------------------
def _expect_prepare(kernel, fused):
    def check(name, d):
        assert d["prepare"] == kernel and d["fused_prepares"] == fused, \
            "%s: prepare kernel %d with %d fused prepares expected, read back %r" % (name, kernel, fused, d)
    return check


def test_prepare_large_k_batches(checker):
    """K = 5000 (> 4096: no k_prepare3, no fused tail) on 480 x 640.  Eight images in one call run k_prepare; five run
    k_prepare2, and so do the two halves of 4 that the blocking host entry makes of 8 images (at slot offset 4)."""
    from fast_slic_b200 import Engine
    H, W, K = 480, 640, 5000
    imgs = _batch(H, W, 8, seed=1300)
    want = _want(checker, _slic(checker, 0.1), imgs, K)
    eng = Engine(H, W, K, 8)
    try:
        p = eng.params(10.0, 0.1, 3, True, 10)
        _check("device B=8", _device(eng, imgs, p), want, _expect_prepare(K_PREPARE, 0))
        _check("host B=8", _host(eng, imgs, p), want, _expect_prepare(K_PREPARE2, 0))
        _check("device B=5", _device(eng, imgs[3:], p), want[3:], _expect_prepare(K_PREPARE2, 0))
        _check("host B=5", _host(eng, imgs[3:], p), want[3:], _expect_prepare(K_PREPARE2, 0))
    finally:
        eng.close()


@pytest.mark.parametrize("K", [4096, 4097])
def test_prepare_k4096_edge(checker, K):
    """K = 4096 is the last K of k_prepare3 and of the prepare fused into the tail of the TMA update launch (one and two
    images); K = 4097 takes k_prepare2 and a k_prepare launch per pass.  The host entry replays a CUDA graph on its
    second call: the read-back is the captured call's."""
    from fast_slic_b200 import Engine
    H, W = 480, 640
    imgs = _batch(H, W, 2, seed=1400 + K)
    want = _want(checker, _slic(checker, 0.1), imgs, K)
    expect = _expect_prepare(K_PREPARE3, 10) if K <= 4096 else _expect_prepare(K_PREPARE2, 0)
    eng = Engine(H, W, K, 2)
    try:
        p = eng.params(10.0, 0.1, 3, True, 10)
        for B in (1, 2):
            _check("device B=%d" % B, _device(eng, imgs[:B], p), want[:B], expect)
            _check("host B=%d" % B, _host(eng, imgs[:B], p), want[:B], expect)
    finally:
        eng.close()


# ---- 4. one-thread-per-pixel kernels past one round of their grid-stride loop ---------------------------------------------
# (id, class, kwargs, checker, float-distance variant): each pass of B = 12 images of 480 x 640 is 1.23 M pixels on the
# update passes and 3.69 M on the full pass, more than one round of a grid capped at 32 CTAs of 256 threads per SM
PIXEL_CASES = [
    ("standard", "SlicRealDist", {}, "real", 0, REAL["standard"]),
    ("l2", "SlicRealDistL2", {}, "real", 1, REAL["l2"]),
    ("noq", "SlicRealDistNoQ", {}, "real", 2, REAL["noq"]),
    ("preemptive", "Slic", dict(preemptive=True, preemptive_thres=0.05), "preemptive", None, PREEMPT),
    ("lsc", "LSC", dict(num_threads=1), "lsc", None, LSC),
    ("euclidean_standard", "SlicRealDist", dict(manhattan_spatial_dist=False), "euclid_real", 0, REAL["standard"]),
    ("euclidean_noq", "SlicRealDistNoQ", dict(manhattan_spatial_dist=False), "euclid_real", 2, REAL["noq"]),
    ("euclidean_preemptive", "Slic", dict(preemptive=True, preemptive_thres=0.05, manhattan_spatial_dist=False),
     "euclid_preemptive", None, PREEMPT),
]


def _pixel_checker(kind, v, checker, euclid, lsc_checker, msf):
    return {"real": lambda: _real(checker, v, msf), "euclid_real": lambda: _real(euclid, v, msf),
            "preemptive": lambda: _slic(checker, msf, preemptive=True, preemptive_thres=0.05),
            "euclid_preemptive": lambda: _slic(euclid, msf, preemptive=True, preemptive_thres=0.05),
            "lsc": lambda: _lsc(lsc_checker, msf)}[kind]()


def _expect_pixels(kernel, H, W, B, full_min_trips=2, upd_min_trips=2):
    def check(name, d):
        _assert_pass(name, d, "update", kernel, _pixels(H, W, B, 3, LAST_REM), min_trips=upd_min_trips)
        if kernel == PREEMPT:  # its full pass is the ordinary one
            assert d["full"]["kernel"] in (TMA, LDG), "%s: preemptive's full pass: %r" % (name, d)
        else:
            _assert_pass(name, d, "full", kernel, _pixels(H, W, B, 1, 0), min_trips=full_min_trips)
        if kernel == LSC:
            assert d["lsc_features_trips"] >= 2, "%s: k_lsc_features ran in one round: %r" % (name, d)
    return check


@pytest.mark.parametrize("case", PIXEL_CASES, ids=[c[0] for c in PIXEL_CASES])
def test_per_pixel_kernels_past_one_trip(checker, euclid, lsc_checker, case):
    """iterate_batch of 12 images with host and device inputs, return_clusters=True, cold and warm start."""
    import fast_slic_b200 as fs
    from fast_slic_b200 import clear_engine_cache, get_engine
    name, cls, kw, kind, v, kernel = case
    H, W, K, B = 480, 640, 400, 12
    imgs = _batch(H, W, B, seed=1500)
    want = _want(checker, _pixel_checker(kind, v, checker, euclid, lsc_checker, 0.25), imgs, K)
    s = getattr(fs, cls)(num_components=K, **kw)
    try:
        host, dev, cl_h, cl_d = [], [], None, None
        t = torch.from_numpy(imgs).cuda()
        for _ in range(2):
            lab, cl_h = s.iterate_batch(imgs, clusters=cl_h, return_clusters=True)
            eng = get_engine(H, W, K, B)
            host.append((lab.view(np.uint16), _pre(eng, B), cl_h.copy(), eng.dispatch()))
        for _ in range(2):
            lab, cl_d = s.iterate_batch(t, clusters=cl_d, return_clusters=True)
            dev.append((lab.cpu().numpy().view(np.uint16), _pre(eng, B), cl_d.cpu().numpy(), eng.dispatch()))
    finally:
        clear_engine_cache()
    expect = _expect_pixels(kernel, H, W, B)
    _check(name + " host", host, want, expect)
    _check(name + " device", dev, want, expect)


@pytest.mark.parametrize("case", [c for c in PIXEL_CASES if c[0] in ("standard", "noq", "preemptive")],
                         ids=lambda c: c[0])
def test_per_pixel_full_pass_1080p(checker, euclid, lsc_checker, case):
    """One 1080 x 1920 image through the class API (Slic*.iterate), cold then warm: the full pass of the float-distance
    kernels is 2.07 M pixels, past one round."""
    import fast_slic_b200 as fs
    from fast_slic_b200 import clear_engine_cache, get_engine
    name, cls, kw, kind, v, kernel = case
    H, W, K = 1080, 1920, 2000
    img = make_image("syn", H, W, seed=1600)
    fn = _pixel_checker(kind, v, checker, euclid, lsc_checker, 0.1)
    expect = _expect_pixels(kernel, H, W, 1, upd_min_trips=1)
    s = getattr(fs, cls)(num_components=K, min_size_factor=0.1, **kw)
    cl = checker.initialize(img, K)
    try:
        for r in range(2):
            got = s.iterate(img).view(np.uint16)
            eng = get_engine(H, W, K, 1)
            pre = _pre(eng, 1)[0]
            wlab, wpre = fn(img, cl)
            where = "%s round %d" % (name, r)
            assert (pre == wpre).all(), "%s: pre-CCA labels differ (%d px)" % (where, int((pre != wpre).sum()))
            assert (got == wlab).all(), "%s: labels differ (%d px)" % (where, int((got != wlab).sum()))
            assert s.slic_model.cluster_array.tobytes() == cl.tobytes(), "%s: Cluster bytes differ" % where
            expect(where, eng.dispatch())
    finally:
        clear_engine_cache()


# ---- 5. the generic kernel past one round ---------------------------------------------------------------------------------
def test_generic_kernel_past_one_trip(checker):
    """2160 x 3840 with K = 300: S = 166, too wide for any spatial-patch pitch of the tile kernels, so both passes run
    k_assign_generic -- 2.76 M pixels per update pass and 8.29 M on the full pass, past one round of its grid."""
    from fast_slic_b200 import Engine
    H, W, K = 2160, 3840, 300
    img = make_image("tiled", H, W, seed=1700)[None]
    want = _want(checker, _slic(checker, 0.25), img, K)

    def expect(name, d):
        _assert_pass(name, d, "update", GENERIC, _pixels(H, W, 1, 3, LAST_REM))
        _assert_pass(name, d, "full", GENERIC, _pixels(H, W, 1, 1, 0))

    eng = Engine(H, W, K, 1)
    try:
        assert eng.S == 166
        p = eng.params(10.0, 0.25, 3, True, 10)
        _check("device", _device(eng, img, p), want, expect)
        _check("host", _host(eng, img, p), want, expect)
    finally:
        eng.close()
