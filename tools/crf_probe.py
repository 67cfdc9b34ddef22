"""Times the SimpleCRF (fast_slic_b200.crf) on the GPU.

1. inference(10) at N = 1600 nodes, C = 21 classes, T in {1, 3, 8} frames: device time from CUDA events around the
   call (1 + 2 x 10 launches), against the plain-C restatement (oracle_crf) on the CPU.
2. A video loop: SlicStream (warm start, one stream) at 1280x720 with K = 1600, push_slic_frame of each frame's clusters
   and labels, set_proba, inference(5) over a sliding window of 3 frames, pop_frame; wall time per frame of each part.

    python tools/crf_probe.py [--frames 30]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def fill(crf, T, N, Cc, rng):
    from crf_cases import random_clusters, random_graph
    for _ in range(T):
        f = crf.push_frame()
        cl = random_clusters(rng, N, "plain")
        f.set_yxmrgb(np.ascontiguousarray(np.stack([cl[n].astype(np.int64) for n in ("y", "x", "num_members", "r",
                                                                                    "g", "b")], 1).astype(np.int32)))
        f.set_connectivity([x[:8] for x in random_graph(rng, N)])
        f.set_proba(rng.dirichlet(np.ones(Cc), N).T.astype(np.float32).copy())
    crf.initialize()


def time_inference(N=1600, Cc=21, reps=20):
    import torch
    from fast_slic_b200.crf import SimpleCRF
    from oracle_crf.crf import Port
    out = {}
    for T in (1, 3, 8):
        rng = np.random.RandomState(T)
        crf = SimpleCRF(Cc, N)
        fill(crf, T, N, Cc, rng)
        crf.inference(10)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ms = []
        for _ in range(reps):
            ev[0].record()
            crf.inference(10)
            ev[1].record()
            torch.cuda.synchronize()
            ms.append(ev[0].elapsed_time(ev[1]))
        # the restatement on the CPU, same sizes
        port = Port(Cc, N)
        rng = np.random.RandomState(T)
        from crf_cases import random_clusters, random_graph, to_csr
        for _ in range(T):
            t = port.push()
            port.set_clusters(t, random_clusters(rng, N, "plain"))
            port.set_connectivity(t, *to_csr([x[:8] for x in random_graph(rng, N)]))
            port.set_proba(t, rng.dirichlet(np.ones(Cc), N).T.astype(np.float32).copy())
        port.initialize()
        t0 = time.perf_counter()
        port.inference(10)
        cpu = (time.perf_counter() - t0) * 1e3
        out["T%d" % T] = dict(gpu_ms_median=float(np.median(ms)), gpu_ms_min=float(np.min(ms)),
                              us_per_iteration=float(np.median(ms)) * 100, cpu_restatement_ms=cpu)
    return out


def video_loop(frames, K=1600, Cc=21, window=3):
    import types
    import torch
    from fast_slic_b200 import SlicModel, SlicStream
    from fast_slic_b200.crf import SimpleCRF
    from oracle.oracle import synthetic_image
    imgs = [synthetic_image(720, 1280, seed=s)[None] for s in range(4)]
    stream = SlicStream(720, 1280, K, batch=1, warm_start=True)
    model = SlicModel(K)
    crf = SimpleCRF(Cc, K)
    rng = np.random.RandomState(0)
    parts = {"slic_stream": [], "push_slic_frame": [], "set_proba": [], "inference5": [], "pop": []}
    for i in range(frames):
        t0 = time.perf_counter()
        stream.submit(imgs[i % 4])
        labels, clusters = stream.collect()
        t1 = time.perf_counter()
        model._clusters = clusters[0]  # what push_slic_frame reads: the model's records and the last label map
        f = crf.push_slic_frame(types.SimpleNamespace(slic_model=model, last_assignment=labels[0]))
        t2 = time.perf_counter()
        f.set_proba(rng.dirichlet(np.ones(Cc), K).T.astype(np.float32).copy())
        f.reset_inferred()
        t3 = time.perf_counter()
        crf.inference(5)
        f.get_inferred()
        t4 = time.perf_counter()
        if crf.num_frames >= window:
            crf.pop_frame()
        t5 = time.perf_counter()
        if i >= 3:
            for k, v in zip(parts, (t1 - t0, t2 - t1, t3 - t2, t4 - t3, t5 - t4)):
                parts[k].append(v * 1e3)
    stream.close()
    torch.cuda.synchronize()
    return {k: float(np.median(v)) for k, v in parts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    a = ap.parse_args()
    import subprocess
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    res = dict(device=torch.cuda.get_device_name(0), card=card, inference10_N1600_C21=time_inference(),
               video_720p_K1600_window3_ms_per_frame=video_loop(a.frames))
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
