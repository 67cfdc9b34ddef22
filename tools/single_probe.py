"""Blocking single-image host call latency, and the latency of the device API on a stream (graph replay from the
second call), on bench.py's workload B (1280x720, K = 1600):  python tools/single_probe.py"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from bench import COMPACTNESS, MAX_ITER, STRIDE, WORKLOADS, synth_images_torch  # noqa: E402
from fast_slic_b200 import CLUSTER_DTYPE, Engine  # noqa: E402

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
