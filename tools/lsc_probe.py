"""The default bench workload (1280x720, K=1600, images resident in HBM) through LSC (fslic_b200_iterate_lsc):

* ms per whole iterate_lsc() step (CUDA events on the launching stream, --steps timed steps after one warm-up);
* the stage split of one timed step (collect_timing=1): cielab_conversion, before_iteration (the feature-mean chains,
  weights, initial centroids), assign (assign + integer update), after_update, full_assign, enforce_connectivity;
* the same split for a single image, where before_iteration is the latency of one serial feature-mean chain;
* parity: image 0 of the last step against the CPU checker (the compiled reference with num_threads=1 where it was
  built, else the restatement), labels and raw Cluster bytes, tolerance 0 -- a mismatch aborts.

python tools/lsc_probe.py [--batch B] [--steps K] -> one JSON line."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from bench import COMPACTNESS, MAX_ITER, STRIDE, WORKLOADS, synth_images_torch
from fast_slic_b200 import Engine
from fast_slic_b200.engine import CLUSTER_DTYPE

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--batch", type=int, default=32)
args = ap.parse_args()
H, W, K, msf = WORKLOADS["B"]
B = args.batch
dev = torch.device("cuda", 0)
eng = Engine(H, W, K, B)
imgs = synth_images_torch(B, H, W, 77, 12.0, dev)
pristine = eng.initialize_clusters(imgs)
lab = torch.empty((B, H, W), dtype=torch.int16, device=dev)
p_fast = eng.params(COMPACTNESS, msf, STRIDE, True, MAX_ITER)
p_timed = eng.params(COMPACTNESS, msf, STRIDE, True, MAX_ITER, collect_timing=1)

cl = pristine.clone()
eng.iterate_lsc(imgs, cl, p_fast, labels=lab)  # warm-up (allocates the LSC scratch, uploads the tables)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
times = []
for _ in range(args.steps):
    cl = pristine.clone()
    e0.record()
    eng.iterate_lsc(imgs, cl, p_fast, labels=lab)
    e1.record()
    e1.synchronize()
    times.append(e0.elapsed_time(e1))

cl_t = pristine.clone()
eng.iterate_lsc(imgs, cl_t, p_timed, labels=torch.empty_like(lab))
stages = eng.stage_ms()
stages.update(eng.lsc_stage_ms())
single = Engine(H, W, K, 1)
cl1 = single.initialize_clusters(imgs[:1].contiguous())
single.iterate_lsc(imgs[:1].contiguous(), cl1, p_timed)
stages1 = single.stage_ms()
stages1.update(single.lsc_stage_ms())

from oracle_lsc.lsc import Port, Ref  # noqa: E402
chk = Ref() if Ref.available() else Port()
img0 = imgs[0].cpu().numpy()
c0 = pristine[0].cpu().numpy().copy().view(CLUSTER_DTYPE).reshape(K)
want = chk.iterate_lsc(img0, c0, MAX_ITER, COMPACTNESS, msf, STRIDE, True)
got = lab[0].cpu().numpy().view(np.uint16)
assert (got == want).all(), "labels of image 0 differ from the checker in %d px" % int((got != want).sum())
assert cl[0].cpu().numpy().tobytes() == c0.tobytes(), "Cluster bytes of image 0 differ from the checker"

times.sort()
print(json.dumps({
    "workload": "%dx%d K=%d batch %d" % (W, H, K, B), "device": torch.cuda.get_device_name(0),
    "checker": type(chk).__module__ + "." + type(chk).__name__,
    "step_ms_median": times[len(times) // 2], "step_ms_min": times[0], "ms_per_image": times[len(times) // 2] / B,
    "stage_ms_batch": {k: round(v, 3) for k, v in stages.items()},
    "stage_ms_single_image": {k: round(v, 3) for k, v in stages1.items()},
    "parity_image0": "bit-exact",
}))
