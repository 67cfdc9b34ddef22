"""Blocking single-image host call latency under a few switches (each in a fresh process):
python tools/single_probe.py            -> table
python tools/single_probe.py --one      -> one measurement with the current environment"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

if "--one" in sys.argv:
    import numpy as np
    import torch
    from bench import COMPACTNESS, MAX_ITER, STRIDE, WORKLOADS, synth_images_torch
    from fast_slic_b200 import CLUSTER_DTYPE, Engine
    H, W, K, msf = WORKLOADS["B"]
    eng = Engine(H, W, K, 1)
    imgs = synth_images_torch(8, H, W, 77, 12.0, torch.device("cuda", 0))
    h = torch.empty((8, 1, H, W, 3), dtype=torch.uint8).pin_memory()
    h.copy_(imgs.view(8, 1, H, W, 3))
    hn = h.numpy()
    pr = eng.initialize_clusters_host(hn[0])
    cl = torch.empty((1, K, 32), dtype=torch.uint8).pin_memory().numpy()
    lab = torch.empty((1, H, W), dtype=torch.int16).pin_memory().numpy()
    p = eng.params(COMPACTNESS, msf, STRIDE, True, MAX_ITER)
    clv = cl.view(CLUSTER_DTYPE).reshape(1, K)
    pr8 = pr.view(np.uint8).reshape(1, K, 32)
    for i in range(20):
        cl[...] = pr8
        eng.iterate_host(hn[i % 8], clv, p, lab)
    ts, sims = [], 0
    for i in range(200):
        cl[...] = pr8
        t0 = time.perf_counter()
        eng.iterate_host(hn[i % 8], clv, p, lab)
        ts.append(time.perf_counter() - t0)
        sims += eng.cca_counters(0)["need_sim"]
    print("mean %.3f ms; calls whose image needed the std::partial_sort replay: %d of 200; per image: %s" % (
        1e3 * sum(ts) / len(ts), sims, ["%.2f" % (1e3 * min(ts[j::8])) for j in range(8)]))
    ts.sort()
    # device API on a side stream (graph replay from the second call)
    st = torch.cuda.Stream()
    d_cl0 = torch.from_numpy(pr8.copy()).cuda()
    d_cl = d_cl0.clone()
    d_lab = torch.empty((1, H, W), dtype=torch.int16, device="cuda")
    with torch.cuda.stream(st):
        for i in range(10):
            d_cl.copy_(d_cl0)
            eng.iterate(imgs[i % 8:i % 8 + 1], d_cl, p, d_lab)
        st.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for i in range(100):
            d_cl.copy_(d_cl0)
            eng.iterate(imgs[i % 8:i % 8 + 1], d_cl, p, d_lab)
        e1.record(st)
        st.synchronize()
    print("host blocking: median %.3f ms  min %.3f  p90 %.3f | device API on a stream: %.3f ms/call" % (
        1e3 * ts[100], 1e3 * ts[0], 1e3 * ts[180], e0.elapsed_time(e1) / 100))
else:
    for env in ({}, {"FSLIC_GRAPH": "0"}, {"FSLIC_ASSIGN": "4"}):
        e = dict(os.environ)
        e.update(env)
        out = subprocess.run([sys.executable, __file__, "--one"], env=e, capture_output=True, text=True)
        print("%-44s %s" % (env or "default", (out.stdout.strip().splitlines() or [out.stderr[-300:]])[-1]))
