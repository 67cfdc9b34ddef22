"""One cached context shared by calls on different streams and entry points, against the checker.

`get_engine` keeps one context per (device, H, W, K); every Slic / SlicRealDist* / LSC / preemptive / debug_mode object
of that shape runs on it, and the context owns all the scratch (Lab image, pre-CCA labels, cluster tables, spatial
patches, LSC tables, connectivity arrays, selection heap).  Consecutive calls must therefore run one after the other on
the device whatever streams they use (capi.cu, CtxOrder).

Overlapping two calls on one context without that order can make the connectivity stage's union-find chase parents two
label maps wrote at once, so the ordering checks never let kernels of two calls overlap on a build without it: the first
call's stream is held by a spin kernel that lasts at least 20 times the second call's measured time plus 20 ms.  Without
the order the second call ends before the first one starts and the check fails on its ordering assertion; with it the
second call waits.  The mixed sequence and the thread test overlap calls for real, so each first passes the first
ordering check and stops there if it fails.

Tolerance: 0 -- labels, pre-CCA labels, Cluster bytes and debug_mode reports are compared exactly.
"""
import threading
import time

import numpy as np
import pytest
import torch

from cases import cca_random_labels, make_image

pytestmark = pytest.mark.gpu

H, W, K = 120, 160, 40
MAX_B = 17  # the largest batch of any call here: the cached context is never rebuilt for a larger one
HELD_B = 3  # images of a device call on a held stream (see _ordered)
KINDS = ("syn", "noise", "blocks")
DEFAULTS = dict(compactness=10.0, min_size_factor=0.25, subsample_stride=3, convert_to_lab=True, max_iter=10)


# ---- the shared context and the checkers ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    """The context every call of this file shares, created first at the largest batch so that no call replaces it."""
    from fast_slic_b200 import get_engine
    return get_engine(H, W, K, MAX_B)


def _assert_same_context(ctx):
    from fast_slic_b200 import base_slic
    assert base_slic._engines.get(("slic", 0, H, W, K)) is ctx, "the shared context was evicted or rebuilt"


@pytest.fixture(scope="module")
def sweep_checkers(checker):
    """(Euclidean checker, its extra iterate keyword arguments, LSC checker), chosen as test_parity_gpu.py chooses them:
    the compiled reference where it was built, else the restatement."""
    from oracle_euclid.euclid import Port as EPort, Ref as ERef
    from oracle_lsc.lsc import Port as LPort, Ref as LRef
    ekw = dict(arch="x64/avx2", num_threads=checker._threads) if ERef.available() else {}
    return ERef() if ERef.available() else EPort(), ekw, LRef() if LRef.available() else LPort()


# A call's class: (name, constructor keyword arguments).  "slic_l2" is Slic(manhattan_spatial_dist=False).
CLASSES = ("slic", "slic_l2", "preemptive", "real_standard", "real_l2", "real_noq", "lsc", "debug")


def _make(cls, args):
    import fast_slic_b200 as fs
    kw = dict(num_components=K, compactness=args["compactness"], min_size_factor=args["min_size_factor"],
              subsample_stride=args["subsample_stride"], convert_to_lab=args["convert_to_lab"])
    if cls == "slic":
        return fs.Slic(**kw)
    if cls == "slic_l2":
        return fs.Slic(manhattan_spatial_dist=False, **kw)
    if cls == "preemptive":
        return fs.Slic(preemptive=True, preemptive_thres=args.get("thres", 0.05), **kw)
    if cls == "lsc":
        return fs.LSC(num_threads=1, **kw)
    if cls == "debug":
        return fs.Slic(debug_mode=True, **kw)
    return {"real_standard": fs.SlicRealDist, "real_l2": fs.SlicRealDistL2, "real_noq": fs.SlicRealDistNoQ}[cls](**kw)


def _expect(checker, sweep_checkers, cls, args, img, cl):
    """(labels, pre-CCA labels) of one call of class `cls` on the checker; `cl` is updated in place (warm start)."""
    euclid, ekw, lsc = sweep_checkers
    a = (args["max_iter"], args["compactness"], args["min_size_factor"], args["subsample_stride"], args["convert_to_lab"])
    if cls in ("slic", "debug"):
        out, _, pre = checker.iterate(img, cl, *a, stages=True)
    elif cls == "slic_l2":
        out, _, pre = euclid.iterate(img, cl, *a, stages=True, **ekw)
    elif cls == "preemptive":
        out, _, pre = checker.iterate(img, cl, *a, stages=True, preemptive=True, preemptive_thres=args.get("thres", 0.05))
    elif cls == "lsc":
        out, st = lsc.iterate_lsc(img, cl, *a, stages=True)
        pre = st["pre"]
    else:
        out, pre = checker.iterate_real(("real_standard", "real_l2", "real_noq").index(cls), img, cl, *a, stages=True)
    return out, pre


def _args(**kw):
    a = dict(DEFAULTS)
    a.update(kw)
    return a


def _images(n, seed):
    return np.stack([make_image(KINDS[(seed + b) % 3], H, W, seed=seed + b) for b in range(n)])


def _u16(x):
    x = x.cpu().numpy() if isinstance(x, torch.Tensor) else x
    return x.view(np.uint16)


def _cluster_bytes(cl):
    return cl.cpu().numpy().tobytes() if isinstance(cl, torch.Tensor) else np.ascontiguousarray(cl).tobytes()


def _check_batch_result(name, checker, sweep_checkers, cls, args, imgs, labels, clusters, pre=None, init=None):
    """Every image of one batch call against the checker: labels, pre-CCA labels (when read back), Cluster bytes.
    `init` are the cluster records the call started from (None: freshly seeded)."""
    labels, pre = _u16(labels), None if pre is None else _u16(pre)
    for b in range(imgs.shape[0]):
        cl = checker.initialize(imgs[b], K) if init is None else init[b].copy()
        want, want_pre = _expect(checker, sweep_checkers, cls, args, imgs[b], cl)
        where = "%s image %d" % (name, b)
        if pre is not None:
            assert (pre[b] == want_pre).all(), "%s: pre-CCA labels differ (%d px)" % (where, int((pre[b] != want_pre).sum()))
        assert (labels[b] == want).all(), "%s: labels differ (%d px)" % (where, int((labels[b] != want).sum()))
        assert _cluster_bytes(clusters[b]) == cl.tobytes(), "%s: Cluster bytes differ" % where


# ---- holding a stream ------------------------------------------------------------------------------------------------
_CYCLES_PER_MS = []


def _cycles_per_ms():
    if not _CYCLES_PER_MS:
        torch.cuda._sleep(1000)  # first launch loads the module
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.cuda._sleep(10_000_000)
        e1.record()
        e1.synchronize()
        _CYCLES_PER_MS.append(10_000_000 / max(e0.elapsed_time(e1), 1e-3))
    return _CYCLES_PER_MS[0]


def _wall_ms(fn):
    """Host wall time of fn() up to an idle device: at least the device time of the work it enqueued."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def _hold(stream, ms):
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(ms * _cycles_per_ms()))


def _ordered(name, x_stream, run_x, run_y, y_stream=None, warm_x=None, warm_y=None):
    """Holds `x_stream`, enqueues X = run_x() there, then Y = run_y() -- on `y_stream`, or as a blocking call when
    `y_stream` is None -- and asserts that Y ended after X.  Returns (X's, Y's) results.

    First `warm_x` (default: X) runs alone on `x_stream` and `warm_y` (default: Y) alone on Y's stream.  That loads
    every kernel the two launch and allocates on both streams before the hold: the first launch of a kernel that is not
    loaded yet can wait for the whole device, which would let X start behind the hold while Y is still being enqueued.
    The hold then lasts 20 times the wall time of `warm_y` plus 20 ms, so without ordering Y ends before X starts.

    A held device call has at most HELD_B images: from 4 images on, the connectivity stage runs part of its tail on the
    context's side stream, and a held call parked there would make a later call's tail wait behind the hold while the
    rest of that call runs -- the two calls would overlap instead of one ending first."""
    with torch.cuda.stream(x_stream):
        _wall_ms(warm_x or run_x)
    with torch.cuda.stream(y_stream or torch.cuda.current_stream()):
        t_y = _wall_ms(warm_y or run_y)
    _hold(x_stream, 20 * t_y + 20)
    with torch.cuda.stream(x_stream):
        rx = run_x()
        ex = torch.cuda.Event(enable_timing=True)
        ex.record()
    if y_stream is None:
        ry = run_y()
        x_done = ex.query()
        torch.cuda.synchronize()
        assert x_done, "%s: the blocking call returned before the call before it on the same context had run" % name
    else:
        with torch.cuda.stream(y_stream):
            ry = run_y()
            ey = torch.cuda.Event(enable_timing=True)
            ey.record()
        torch.cuda.synchronize()
        dt = ex.elapsed_time(ey)
        assert dt > 0, "%s: the second call ended %.3f ms before the first one on the same context" % (name, -dt)
    return rx, ry


def _device_batch(cls, args, x, ctx):
    """Device iterate_batch of class `cls` on the current stream, then its pre-CCA labels read back on that stream."""
    lab, cl = _make(cls, args).iterate_batch(x, max_iter=args["max_iter"], return_clusters=True)
    return lab, cl, ctx.debug_stages(x.shape[0])[1]


def _upload(imgs):
    x = torch.from_numpy(imgs).cuda()
    torch.cuda.synchronize()  # inputs are complete before any held or foreign stream reads them
    return x


def _gate(checker, sweep_checkers, ctx):
    """Ordering check (a) 1, which the overlapping tests need before they may overlap anything."""
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a1, a2 = _args(), _args(compactness=20.0, min_size_factor=0.1)
    i1, i2 = _images(HELD_B, 100), _images(5, 110)
    x1, x2 = _upload(i1), _upload(i2)
    rx, ry = _ordered("device iterate_batch on two streams", s1, lambda: _device_batch("slic", a1, x1, ctx),
                      lambda: _device_batch("slic", a2, x2, ctx), y_stream=s2)
    _check_batch_result("first call", checker, sweep_checkers, "slic", a1, i1, *rx)
    _check_batch_result("second call", checker, sweep_checkers, "slic", a2, i2, *ry)


# ---- (a) ordering: X on a held stream, then Y ------------------------------------------------------------------------
def test_order_device_batches_on_two_streams(checker, sweep_checkers, ctx):
    """Device iterate_batch of three images on one stream, then a call of five images (the connectivity tail split
    onto the side stream) with other parameters on another stream."""
    _gate(checker, sweep_checkers, ctx)
    _assert_same_context(ctx)


def test_order_graph_replays_on_two_streams(checker, ctx):
    """Engine.iterate of two images with fixed buffers: captured into a CUDA graph on one stream, then one replay on
    the held stream and one on another stream.  Every call warm-starts from the clusters the one before wrote, so the
    last replay's labels and clusters are the checker's sixth iterate of the chain."""
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    imgs = [_images(2, 200 + 10 * t) for t in range(6)]
    xs = [_upload(i) for i in imgs]
    p = ctx.params(10.0, 0.1, 3, True, 10)
    with torch.cuda.stream(s1):
        cl = ctx.initialize_clusters(xs[0])
        lab = torch.empty((2, H, W), dtype=torch.int16, device="cuda")
    captures0, replays0 = ctx.graph_counts()
    with torch.cuda.stream(s1):
        ctx.iterate(xs[0], cl, p, lab)
        ctx.iterate(xs[1], cl, p, lab)  # the same key again: captured
    torch.cuda.synchronize()
    assert ctx.graph_counts()[0] == captures0 + 1, "the second call was not captured"

    def replay(x):
        ctx.iterate(x, cl, p, lab)
        return ctx.debug_stages(2)[1]

    _, pre = _ordered("graph replays on two streams", s1, lambda: replay(xs[4]), lambda: replay(xs[5]), y_stream=s2,
                      warm_x=lambda: replay(xs[2]), warm_y=lambda: replay(xs[3]))
    captures, replays = ctx.graph_counts()
    assert captures == captures0 + 1 and replays >= replays0 + 4, "the calls did not replay the graph"
    for b in range(2):
        c0 = checker.initialize(imgs[0][b], K)
        for t in range(6):
            want, _, want_pre = checker.iterate(imgs[t][b], c0, 10, 10.0, 0.1, 3, True, stages=True)
        assert (_u16(pre)[b] == want_pre).all(), "image %d: pre-CCA labels differ" % b
        assert (_u16(lab)[b] == want).all(), "image %d: labels differ" % b
        assert cl[b].cpu().numpy().tobytes() == c0.tobytes(), "image %d: Cluster bytes differ" % b
    _assert_same_context(ctx)


def test_order_device_then_host_paths(checker, sweep_checkers, ctx):
    """Device iterate_batch on the held legacy default stream, then each host path, which runs on the context's own
    non-blocking streams: Slic.iterate of one numpy image (the plain host path, timed), iterate_batch of two numpy
    images (the replayed host graph) and of 17 (the two-lane path)."""
    from fast_slic_b200 import Slic
    default = torch.cuda.default_stream()
    a = _args(min_size_factor=0.1)
    one = make_image("syn", H, W, seed=301)
    two, many = _images(2, 310), _images(MAX_B, 320)
    Slic(num_components=K, min_size_factor=0.1).iterate_batch(two)  # the host graph of two images is captured here: the calls below replay it
    replays0 = ctx.graph_counts()[1]
    host_calls = [
        ("Slic.iterate (host)", lambda: (lambda s: (s.iterate(one)[None], s.slic_model.cluster_array[None]))(
            Slic(num_components=K, min_size_factor=0.1)), one[None]),
        ("iterate_batch of 2 numpy images (host graph)",
         lambda: Slic(num_components=K, min_size_factor=0.1).iterate_batch(two, return_clusters=True), two),
        ("iterate_batch of 17 numpy images (two lanes)",
         lambda: Slic(num_components=K, min_size_factor=0.1).iterate_batch(many, return_clusters=True), many),
    ]
    for t, (name, run_y, y_imgs) in enumerate(host_calls):
        ix = _images(HELD_B, 330 + 10 * t)
        x = _upload(ix)

        def run_y_pre():
            lab, cl = run_y()
            return lab, cl, ctx.debug_stages(y_imgs.shape[0])[1]

        rx, ry = _ordered("device call, then " + name, default, lambda: _device_batch("slic", _args(), x, ctx), run_y_pre)
        _check_batch_result(name + ": device call", checker, sweep_checkers, "slic", _args(), ix, *rx)
        _check_batch_result(name, checker, sweep_checkers, "slic", a, y_imgs, *ry)
    assert ctx.graph_counts()[1] >= replays0 + 2, "the two-image host calls did not replay the graph"
    _assert_same_context(ctx)


def test_order_device_then_real_dist_numpy(checker, sweep_checkers, ctx):
    """Device iterate_batch on a held stream, then SlicRealDist.iterate of a numpy image, which runs on the current
    torch stream (here the legacy default stream) and blocks."""
    from fast_slic_b200 import SlicRealDist
    s1 = torch.cuda.Stream()
    ix = _images(HELD_B, 400)
    x = _upload(ix)
    img = make_image("syn", H, W, seed=410)

    def run_y():
        s = SlicRealDist(num_components=K)
        lab = s.iterate(img)
        return lab[None], s.slic_model.cluster_array[None], ctx.debug_stages(1)[1]

    rx, ry = _ordered("device call, then SlicRealDist.iterate", s1, lambda: _device_batch("slic", _args(), x, ctx), run_y)
    _check_batch_result("device call", checker, sweep_checkers, "slic", _args(), ix, *rx)
    _check_batch_result("SlicRealDist.iterate", checker, sweep_checkers, "real_standard", _args(), img[None], *ry)
    _assert_same_context(ctx)


def test_order_device_then_debug_stages(checker, sweep_checkers, ctx):
    """Device iterate_batch on a held stream, then Engine.debug_stages on another stream: it returns that call's Lab
    image and pre-CCA labels, not the previous call's."""
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    ix = _images(3, 500)
    x, other = _upload(ix), _upload(_images(3, 510))
    rx, (quad, pre) = _ordered("device call, then debug_stages", s1,
                               lambda: _make("slic", _args()).iterate_batch(x, return_clusters=True),
                               lambda: ctx.debug_stages(3), y_stream=s2,
                               warm_x=lambda: _device_batch("slic", _args(), other, ctx))  # leaves other labels behind
    _check_batch_result("device call", checker, sweep_checkers, "slic", _args(), ix, rx[0], rx[1], pre)
    for b in range(3):
        _, want_quad, _ = checker.iterate(ix[b], checker.initialize(ix[b], K), stages=True)
        assert (quad[b].cpu().numpy() == want_quad).all(), "image %d: Lab image differs" % b
    _assert_same_context(ctx)


def test_order_lsc_table_rebuild(checker, sweep_checkers, ctx):
    """LSC iterate_batch on a held stream, then on another stream with another compactness: the second call rebuilds
    the context's LSC feature table, which the first one reads."""
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a1, a2 = _args(compactness=10.0), _args(compactness=30.0, min_size_factor=0.1)
    i1, i2 = _images(3, 600), _images(3, 610)
    x1, x2 = _upload(i1), _upload(i2)
    rx, ry = _ordered("LSC on two streams", s1, lambda: _device_batch("lsc", a1, x1, ctx),
                      lambda: _device_batch("lsc", a2, x2, ctx), y_stream=s2)
    _check_batch_result("first LSC call", checker, sweep_checkers, "lsc", a1, i1, *rx)
    _check_batch_result("second LSC call", checker, sweep_checkers, "lsc", a2, i2, *ry)
    _assert_same_context(ctx)


def test_order_connectivity_only_context(checker, ctx):
    """Engine(cca_only=True).enforce_connectivity on a held stream, then on another stream with other label maps."""
    from fast_slic_b200 import Engine
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    eng = Engine(H, W, max_batch=3, cca_only=True)
    try:
        maps = [np.stack([cca_random_labels(H, W, 30, 700 + 10 * t + b) for b in range(3)]) for t in range(4)]
        thres = (20, 5, 20, 5)
        ts = [_upload(m) for m in maps]
        run = [lambda t=t: eng.enforce_connectivity(ts[t], 30, thres[t]) for t in range(4)]
        _ordered("enforce_connectivity on two streams", s1, run[0], run[1], y_stream=s2, warm_x=run[2], warm_y=run[3])
        for t in range(2):
            for b in range(3):
                want = checker.enforce_connectivity(maps[t][b].view(np.uint16), 30, thres[t])
                got = _u16(ts[t][b])
                assert (got == want).all(), "call %d map %d: %d px differ" % (t, b, int((got != want).sum()))
    finally:
        eng.close()
    _assert_same_context(ctx)


# ---- (b) a seeded mixed sequence ---------------------------------------------------------------------------------
ENTRIES = ("numpy_iterate", "numpy_batch", "tensor_default", "tensor_s1", "tensor_s2", "host_async")


def _mixed_steps(seed, n):
    """[(class, entry point, batch, arguments)] drawn from a seeded generator; a forced pair of identical two-image
    host batches with their own compactness guarantees one graph capture and one replay."""
    rng = np.random.RandomState(seed)
    steps = []
    while len(steps) < n:
        cls = CLASSES[rng.randint(len(CLASSES))]
        entry = ENTRIES[rng.randint(len(ENTRIES))]
        if cls == "debug":
            entry = "numpy_iterate"  # debug_mode reports belong to iterate()
        if entry == "host_async" and (cls not in ("slic", "slic_l2") or (steps and steps[-1][1] == "host_async")):
            entry = "numpy_batch"  # the host entry points serve the integer Slic path; one pending batch at a time
        batch = 1 if entry == "numpy_iterate" else (1, 2, 3, 5, MAX_B)[rng.randint(5)]
        args = _args(compactness=float((5, 10, 20, 40)[rng.randint(4)]), subsample_stride=int((1, 2, 3, 5)[rng.randint(4)]),
                     max_iter=int((0, 1, 5, 10)[rng.randint(4)]), min_size_factor=float((0.0, 0.1, 0.25, 0.5)[rng.randint(4)]),
                     convert_to_lab=bool(rng.randint(2)), thres=float((0.05, 0.1)[rng.randint(2)]))
        steps.append((cls, entry, batch, args))
    forced = ("slic", "numpy_batch", 2, _args(compactness=13.0))
    k = n // 3
    steps[k:k] = [forced, forced]
    if steps[-1][1] == "host_async":
        steps.append(("slic", "numpy_batch", 1, _args()))
    return steps


def test_mixed_sequence_on_one_context(checker, sweep_checkers, ctx):
    """About 24 calls of every class and entry point on the one context with no synchronisation except where an API
    blocks: numpy iterate (cold, then warm), numpy iterate_batch, tensor iterate_batch on the default stream and on two
    other streams, Engine.iterate_host_async waited for only after the next call.  Every call's labels, pre-CCA labels
    (read back behind it) and Cluster bytes against the checker; debug_mode reports against the same call on a fresh
    context."""
    from fast_slic_b200 import CLUSTER_DTYPE, Engine
    _gate(checker, sweep_checkers, ctx)
    steps = _mixed_steps(2024, 22)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    streams = {"tensor_default": torch.cuda.default_stream(), "tensor_s1": s1, "tensor_s2": s2}
    inputs = [_images(b, 1000 + 20 * i) for i, (_, _, b, _) in enumerate(steps)]
    device_inputs = {i: torch.from_numpy(inputs[i]).cuda() for i, s in enumerate(steps) if s[1] in streams}
    pinned = {}
    for i, (_, entry, b, _) in enumerate(steps):
        if entry == "host_async":
            img = torch.from_numpy(inputs[i]).pin_memory()
            pinned[i] = (img, torch.empty((b, K, 32), dtype=torch.uint8).pin_memory(),
                         torch.empty((b, H, W), dtype=torch.int16).pin_memory())
    torch.cuda.synchronize()
    captures0, replays0 = ctx.graph_counts()
    results, reports, waiting = [], [], None
    for i, (cls, entry, b, args) in enumerate(steps):
        if entry == "numpy_iterate":
            s = _make(cls, args)
            for run in ("cold", "warm"):
                lab = s.iterate(inputs[i][0], max_iter=args["max_iter"])
                results.append((i, run, lab[None], s.slic_model.cluster_array.copy()[None], ctx.debug_stages(1)[1]))
                if cls == "debug":
                    reports.append((i, run, s.slic_model.last_recorder_report))
        elif entry == "numpy_batch":
            lab, cl = _make(cls, args).iterate_batch(inputs[i], max_iter=args["max_iter"], return_clusters=True)
            results.append((i, None, lab, cl, ctx.debug_stages(b)[1]))
        elif entry in streams:
            with torch.cuda.stream(streams[entry]):
                results.append((i, None) + _device_batch(cls, args, device_inputs[i], ctx))
        else:
            img, cl, lab = pinned[i]
            cl.numpy()[...] = ctx.initialize_clusters_host(inputs[i]).view(np.uint8).reshape(b, K, 32)
            p = ctx.params(args["compactness"], args["min_size_factor"], args["subsample_stride"], args["convert_to_lab"],
                           args["max_iter"])
            ctx.iterate_host_async(img.numpy(), cl.numpy().view(CLUSTER_DTYPE).reshape(b, K), p, lab.numpy(),
                                   manhattan_spatial_dist=cls == "slic")
            results.append((i, None, lab, cl, ctx.debug_stages(b)[1]))
        if waiting is not None:  # the pending host batch of the previous step, after this step's call
            ctx.wait()
            waiting = None
        if entry == "host_async":
            waiting = i
    torch.cuda.synchronize()
    captures, replays = ctx.graph_counts()
    assert captures > captures0 and replays > replays0, "no CUDA graph was captured and replayed: %r -> %r" % (
        (captures0, replays0), (captures, replays))

    warm = {}
    for i, run, lab, cl, pre in results:
        cls, entry, b, args = steps[i]
        name = "step %d (%s, %s, B=%d, %r)%s" % (i, cls, entry, b, args, "" if run is None else " " + run)
        init = None
        if run == "warm":
            init = warm[i]
        elif run == "cold":
            c0 = checker.initialize(inputs[i][0], K)
            _expect(checker, sweep_checkers, cls, args, inputs[i][0], c0)
            warm[i] = c0[None]
        if entry == "host_async":
            cl = cl.numpy().view(CLUSTER_DTYPE).reshape(b, K)
        _check_batch_result(name, checker, sweep_checkers, cls, args, inputs[i], lab, cl, pre, init)
    for i, run, report in reports:
        args = steps[i][3]
        assert report == _fresh_report(checker, sweep_checkers, Engine, inputs[i][0], args, warm=run == "warm"), \
            "step %d %s: the debug_mode report differs from the same call on a fresh context" % (i, run)
    _assert_same_context(ctx)


def _fresh_report(checker, sweep_checkers, Engine, img, args, warm):
    """The debug_mode report of Slic(debug_mode=True).iterate(img) (cold) or of its second call (warm), on a context of
    its own."""
    eng = Engine(H, W, K, 1)
    try:
        cl = checker.initialize(img, K)
        if warm:
            _expect(checker, sweep_checkers, "slic", args, img, cl)
        x = torch.from_numpy(img[None]).cuda()
        d_cl = torch.from_numpy(cl.view(np.uint8).reshape(1, K, 32).copy()).cuda()
        p = eng.params(args["compactness"], args["min_size_factor"], args["subsample_stride"], args["convert_to_lab"],
                       args["max_iter"], collect_timing=1)
        eng.set_trace(True)
        eng.iterate(x, d_cl, p)
        return eng.recorder_report(0)
    finally:
        eng.close()


# ---- (c) two threads -----------------------------------------------------------------------------------------------
def test_two_threads_own_streams(checker, sweep_checkers, ctx):
    """Two host threads, each with its own torch stream, run tensor iterate_batch calls with different images and
    compactness on the one context; one thread also runs numpy Slic.iterate calls.  Every result against the checker;
    pre-CCA labels are read back under the context's lock, behind the call they belong to."""
    from fast_slic_b200 import Slic
    _gate(checker, sweep_checkers, ctx)
    plans = [[(c, _images(b, 2000 + 100 * t + 10 * j)) for j, (c, b) in enumerate(((10.0, 5), (20.0, 3), (5.0, 2), (40.0, 5)))]
             for t in range(2)]
    singles = [make_image(KINDS[j % 3], H, W, seed=2500 + j) for j in range(3)]
    inputs = [[_upload(imgs) for _, imgs in plan] for plan in plans]
    out = [[], []]
    single_out = []
    errors = []

    def work(t):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for j, (c, imgs) in enumerate(plans[t]):
                    with ctx.lock:
                        lab, cl = Slic(num_components=K, compactness=c).iterate_batch(inputs[t][j], return_clusters=True)
                        out[t].append((lab, cl, ctx.debug_stages(imgs.shape[0])[1]))
                    if t == 1 and j < len(singles):
                        s = Slic(num_components=K, compactness=c)
                        single_out.append((c, s.iterate(singles[j]), s.slic_model.cluster_array.copy()))
            st.synchronize()
        except Exception as e:  # noqa: BLE001
            errors.append("thread %d: %r" % (t, e))

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    torch.cuda.synchronize()
    assert not errors, errors
    for t in range(2):
        for j, (c, imgs) in enumerate(plans[t]):
            _check_batch_result("thread %d call %d" % (t, j), checker, sweep_checkers, "slic", _args(compactness=c), imgs,
                                *out[t][j])
    for j, (c, lab, cl) in enumerate(single_out):
        _check_batch_result("thread 1 numpy iterate %d" % j, checker, sweep_checkers, "slic", _args(compactness=c),
                            singles[j][None], lab[None], cl[None])
    _assert_same_context(ctx)
