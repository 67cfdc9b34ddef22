"""The default bench workload (1280x720, K=1600, batch 32, images resident in HBM) with the Manhattan and the Euclidean
spatial term, alternating the two settings on one context so both see the same card state:

* per-launch time of the fused assign+update kernel (collect_timing=2, CUDA events around each launch);
* ms per whole iterate() step (CUDA events on the launching stream, --steps steps per setting and round);
* parity: image 0 of the last step of each setting against the CPU checker of that setting (the compiled reference
  where it was built, else the restatement), labels and raw Cluster bytes, tolerance 0 -- a mismatch aborts.

python tools/spatial_dist_probe.py [--rounds N] [--steps K] -> one JSON line."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from bench import COMPACTNESS, MAX_ITER, STRIDE, WORKLOADS, synth_images_torch
from fast_slic_b200 import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--batch", type=int, default=32)
args = ap.parse_args()
H, W, K, msf = WORKLOADS["B"]
B = args.batch
dev = torch.device("cuda", 0)
eng = Engine(H, W, K, B)
imgs = synth_images_torch(B, H, W, 77, 12.0, dev)
pristine = eng.initialize_clusters(imgs)
cl = pristine.clone()
lab = torch.empty((B, H, W), dtype=torch.int16, device=dev)
p_timed = eng.params(COMPACTNESS, msf, STRIDE, True, MAX_ITER, collect_timing=2)
p_fast = eng.params(COMPACTNESS, msf, STRIDE, True, MAX_ITER)
SETTINGS = (True, False)
per_launch = {m: [] for m in SETTINGS}
step_ms = {m: [] for m in SETTINGS}
impl = {}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for r in range(args.rounds + 1):  # round 0 warms up
    for m in SETTINGS:
        cl.copy_(pristine)
        eng.iterate(imgs, cl, p_timed, lab, manhattan_spatial_dist=m)
        ms, n = eng.assign_kernel_time()
        impl[m] = eng.assign_impl()
        e0.record()
        for _ in range(args.steps):
            cl.copy_(pristine)  # every step is a cold start
            eng.iterate(imgs, cl, p_fast, lab, manhattan_spatial_dist=m)
        e1.record()
        e1.synchronize()
        if r:
            per_launch[m].append(ms / n)
            step_ms[m].append(e0.elapsed_time(e1) / args.steps)

parity = {}
img0 = np.ascontiguousarray(imgs[0].cpu().numpy())
for m in SETTINGS:
    cl.copy_(pristine)
    eng.iterate(imgs, cl, p_fast, lab, manhattan_spatial_dist=m)
    got_lab, got_cl = lab[0].cpu().numpy().view(np.uint16), cl[0].cpu().numpy()
    if m:
        from oracle.oracle import Port, Ref
    else:
        from oracle_euclid.euclid import Port, Ref
    use_ref = Ref.available()
    chk = Ref() if use_ref else Port()
    c0 = chk.initialize(img0, K)
    kw = dict(arch="x64/avx2", num_threads=8) if use_ref else {}
    want = chk.iterate(img0, c0, MAX_ITER, COMPACTNESS, msf, STRIDE, True, **kw)
    ok = bool((got_lab == want).all()) and got_cl.tobytes() == c0.view(np.uint8).tobytes()
    assert ok, "setting manhattan=%s: image 0 differs from the CPU checker" % m
    parity[m] = "reference" if use_ref else "port"

name = {True: "manhattan", False: "euclidean"}
mp = B * H * W / 1e6
print(json.dumps({"workload": "%dx%d K=%d, batch %d, images in HBM, %s" % (W, H, K, B, torch.cuda.get_device_name(0)),
                  "rounds": args.rounds, "steps_per_round": args.steps,
                  **{name[m]: {"assign_ms_per_launch_median": float(np.median(per_launch[m])),
                               "assign_ms_per_launch_min": float(np.min(per_launch[m])),
                               "ms_per_step_median": float(np.median(step_ms[m])),
                               "megapixels_per_s_median": mp / (float(np.median(step_ms[m])) / 1e3),
                               "assign_impl": impl[m], "parity_checked_against": parity[m]} for m in SETTINGS}}))
