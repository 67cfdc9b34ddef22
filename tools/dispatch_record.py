"""Launch decisions and outputs of a fixed matrix of iterate and enforce_connectivity calls, as JSON, for one build of
the library:

    python tools/dispatch_record.py path/to/libfslic_b200.so out.json

For every configuration it records launches_last_iterate, dispatch() (with the connectivity stage's decisions),
graph_counts() and SHA-256 digests of the labels and clusters; for the connectivity-only calls the stage's decisions,
the per-image counters and the label digest.  Two builds that make the same launch decisions and
compute the same results write identical files, so a host-side change is checked with a diff of two runs (one process
per library: the binding loads one library per process)."""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import cca_cases  # noqa: E402
from bench import synth_images_torch  # noqa: E402
from fast_slic_b200 import _lib  # noqa: E402


def digest(a):
    if isinstance(a, torch.Tensor):
        a = a.cpu().numpy()
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def record(eng, labels, clusters, **extra):
    r = {"launches": eng.launches_last_iterate(), "dispatch": eng.dispatch(), "graph_counts": list(eng.graph_counts()),
         "labels": digest(labels), "clusters": digest(clusters)}
    r.update(extra)
    return r


class Env:
    """Environment switches for the calls (or engine creation) inside the block"""

    def __init__(self, **kv):
        self.kv = kv

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kv}
        os.environ.update(self.kv)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def main(lib_path, out_path):
    _lib.LIB_PATH = os.path.abspath(lib_path)
    from fast_slic_b200 import Engine
    dev = torch.device("cuda", 0)
    out = {}
    imgs = {}

    def images(H, W, B):
        if (H, W) not in imgs:
            imgs[(H, W)] = synth_images_torch(40, H, W, 1234, 12.0, dev)
        return imgs[(H, W)][:B].contiguous()

    def device_run(name, H, W, K, B, kind="u16", env=None, manhattan=True, trace=False, **pk):
        with Env(**(env or {})):
            eng = Engine(H, W, K, B)
            im = images(H, W, B)
            cl = eng.initialize_clusters(im)
            p = eng.params(**pk)
            if trace:
                eng.set_trace(True)
            if kind == "u16":
                lab = eng.iterate(im, cl, p, manhattan_spatial_dist=manhattan)
            elif kind == "preemptive":
                lab = eng.iterate_preemptive(im, cl, p, 0.5, manhattan_spatial_dist=manhattan)
            elif kind == "lsc":
                lab = eng.iterate_lsc(im, cl, p)
            else:
                lab = eng.iterate_real(kind, im, cl, p, manhattan_spatial_dist=manhattan)
            torch.cuda.synchronize()
            extra = {}
            if trace:
                s = eng.trace_snapshots(0)
                extra["trace"] = [digest(s["assignment"]), digest(s["min_dists"]), digest(s["clusters"])]
                eng.set_trace(False)
            if pk.get("collect_timing", 0) >= 2:
                extra["assign_kernel_launches"] = eng.assign_kernel_time()[1]
            out[name] = record(eng, lab, cl, **extra)
            eng.close()

    # the u16 path: TMA (W % 8 == 0, stride 3), LDG (W % 8 != 0), generic (S > 160: no patch in smem)
    for B in (1, 2, 8, 32):
        device_run("tma_b%d" % B, 240, 320, 300, B)
        device_run("generic_b%d" % B, 400, 400, 4, B)
    device_run("w_mod8_b1", 241, 323, 300, 1)
    device_run("w_mod8_b8", 241, 323, 300, 8)
    device_run("stride1_b2", 240, 320, 300, 2, subsample_stride=1)
    device_run("stride5_b2", 240, 320, 300, 2, subsample_stride=5)
    device_run("euclid_b8", 240, 320, 300, 8, manhattan=False)
    # bookkeeping kernels: K > 4096 takes k_prepare2 below 8 images and k_prepare from 8
    device_run("bigk_b1", 480, 640, 6000, 1)
    device_run("bigk_b8", 480, 640, 6000, 8)
    for v in ("standard", "l2", "noq"):
        for man in (True, False):
            for B in (1, 8):
                device_run("real_%s_%s_b%d" % (v, "man" if man else "euc", B), 240, 320, 300, B, kind=v, manhattan=man)
    for B in (1, 8):
        device_run("preemptive_b%d" % B, 240, 320, 300, B, kind="preemptive")
        device_run("lsc_b%d" % B, 240, 320, 300, B, kind="lsc")
    device_run("traced_u16_b2", 240, 320, 300, 2, trace=True, max_iter=4)
    device_run("traced_preemptive_b2", 240, 320, 300, 2, kind="preemptive", trace=True, max_iter=4)
    device_run("traced_real_noq_b2", 240, 320, 300, 2, kind="noq", trace=True, max_iter=4)
    device_run("traced_lsc_b2", 240, 320, 300, 2, kind="lsc", trace=True, max_iter=4)
    for t in (1, 2):
        device_run("timing%d_b2" % t, 240, 320, 300, 2, collect_timing=t)
        device_run("timing%d_b8" % t, 240, 320, 300, 8, collect_timing=t)
        device_run("timing%d_lsc_b2" % t, 240, 320, 300, 2, kind="lsc", collect_timing=t)

    # graph replay of the device entry point: the second identical call captures, the third replays
    eng = Engine(240, 320, 300, 2)
    im = images(240, 320, 2)
    cl0 = eng.initialize_clusters(im)
    cl = cl0.clone()
    lab = torch.empty((2, 240, 320), dtype=torch.int16, device=dev)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for i in range(3):
            cl.copy_(cl0)
            eng.iterate(im, cl, eng.params(), lab)
            st.synchronize()
            out["graph_call%d" % i] = record(eng, lab, cl)
    eng.close()

    # host entry points: graph (< 4 images), plain, split (8+), two lanes (16..64), chunked (> 32 or FSLIC_HOST_CHUNK)
    def host_run(name, B, calls=1, env=None, is_async=False, collect_timing=0):
        with Env(**(env or {})):
            eng = Engine(240, 320, 300, B)
            im = images(240, 320, B).cpu().numpy()
            cl0 = eng.initialize_clusters_host(im)
            for i in range(calls):
                cl = cl0.copy()
                lab = np.empty((B, 240, 320), np.int16)
                p = eng.params(collect_timing=collect_timing)
                if is_async:
                    eng.iterate_host_async(im, cl, p, lab)
                    eng.wait()
                else:
                    eng.iterate_host(im, cl, p, lab)
                out["%s_call%d" % (name, i)] = record(eng, lab, cl)
                if collect_timing:  # which of the connectivity stage's sub-sections were timed
                    out["%s_call%d" % (name, i)]["cca_stage_ms"] = sorted(k for k, v in eng.cca_stage_ms().items() if v > 0)
            eng.close()

    for B in (1, 3, 8, 16, 32, 40):
        host_run("host_b%d" % B, B, calls=2)
    host_run("host_timing_b2", 2, collect_timing=1)
    host_run("host_chunk4_b8", 8, env={"FSLIC_HOST_CHUNK": "4"})
    host_run("host_chunk8_b24", 24, env={"FSLIC_HOST_CHUNK": "8"})
    host_run("host_async_b8", 8, is_async=True)
    host_run("host_async_b24", 24, is_async=True)
    host_run("host_async_b2", 2, calls=2, is_async=True)

    # the connectivity stage alone: maps whose K-th largest area is tied (the std::partial_sort replay) beside maps
    # with fewer candidates than K; one stream (B = 1), the settled images' tail on the side stream (B = 4), sub-batches
    # of 3 (B = 8), whose counters hold the last sub-batch
    ties = [cca_cases.random_rect_grid(240, 320, [1, 2], [1, 2, 3], seed) for seed in range(8)]
    K = cca_cases.k_for(cca_cases.components(ties[0])[2], 1, True, 4)
    maps = np.stack([ties[i] if i % 2 == 0 else cca_cases.bands(240, 320, [50 + i, 60]) for i in range(8)])

    def cca_run(name, B, sub_batch=None):
        with Env(**({"FSLIC_CCA_BATCH": str(sub_batch)} if sub_batch else {})):
            eng = Engine(240, 320, max_batch=B, cca_only=True)
            lab = torch.from_numpy(maps[:B].view(np.int16)).to(dev)
            eng.enforce_connectivity(lab, K, 1)
            torch.cuda.synchronize()
            out[name] = {"cca": eng.dispatch()["cca"], "labels": digest(lab),
                         "counters": [eng.cca_counters(i) for i in range(sub_batch or B)]}
            eng.close()

    cca_run("cca_b1", 1)
    cca_run("cca_b4", 4)
    cca_run("cca_b8_sub3", 8, sub_batch=3)

    with open(out_path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("%d configurations -> %s" % (len(out), out_path))


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    main(sys.argv[1], sys.argv[2])
