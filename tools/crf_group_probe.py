"""Times the temporal CRFs of B video streams driven one by one against the same CRFs driven as one SimpleCRFGroup.

Workload: B = 32 streams, warm-started Slic.iterate_batch on the GPU at 1280x720 with K = 1600 (image b of each batch
is the next frame of stream b), C = 21 class probabilities per superpixel, inference(5) over a sliding window of 3
frames, the newest frame's q read into a cuda tensor, and pop_frame.  Every step feeds both of:

  loop   32 device-fed SimpleCRFs, each called on its own: push_label_frames(labels[b], clusters[b]),
         set_proba, reset_inferred, inference(5), get_inferred(out=), pop_frame
  group  32 more SimpleCRFs as one SimpleCRFGroup: the same calls, once for all members

from the same SLIC output, alternating within each step.  Each part is followed by a device synchronisation, so its
wall time includes the GPU work it enqueued.  Reports the median per step and per part, and the card's name and power
limit; exits non-zero unless every member's last q is bit-identical between the two runs.

    python tools/crf_group_probe.py [--frames 30] [--streams 32]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PARTS = ("push", "set_proba_reset", "inference5_get", "pop")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--streams", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    from fast_slic_b200 import Slic
    from fast_slic_b200.crf import SimpleCRF, SimpleCRFGroup
    from oracle.oracle import synthetic_image
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    B, K, Cc, window = a.streams, 1600, 21, 3
    pool = torch.from_numpy(np.stack([synthetic_image(720, 1280, seed=s) for s in range(8)])).cuda()
    rng = np.random.RandomState(0)
    probas = [torch.from_numpy(rng.dirichlet(np.ones(Cc), (B, K)).transpose(0, 2, 1).astype(np.float32).copy()).cuda()
              for _ in range(4)]
    slic = Slic(num_components=K)
    loop = [SimpleCRF(Cc, K) for _ in range(B)]
    group = SimpleCRFGroup([SimpleCRF(Cc, K) for _ in range(B)])
    q_loop = torch.empty(B, Cc, K, device="cuda")
    q_group = torch.empty(B, Cc, K, device="cuda")
    ms = {mode: {k: [] for k in PARTS + ("step",)} for mode in ("loop", "group")}
    slic_ms = []
    clusters = None
    for i in range(a.frames + a.warmup):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        images = pool[torch.tensor([(i + b) % 8 for b in range(B)], device="cuda")]
        labels, clusters = slic.iterate_batch(images, clusters=clusters, return_clusters=True)
        torch.cuda.synchronize()
        if i >= a.warmup:
            slic_ms.append((time.perf_counter() - t0) * 1e3)
        proba = probas[i % 4]
        for mode in ("loop", "group"):
            t = [time.perf_counter()]

            def mark():
                torch.cuda.synchronize()
                t.append(time.perf_counter())

            if mode == "loop":
                frames = [crf.push_label_frames(labels[b], clusters[b]) for b, crf in enumerate(loop)]
                mark()
                for b, f in enumerate(frames):
                    f.set_proba(proba[b])
                    f.reset_inferred()
                mark()
                for b, (crf, f) in enumerate(zip(loop, frames)):
                    crf.inference(5)
                    f.get_inferred(out=q_loop[b])
                mark()
                if loop[0].num_frames >= window:
                    for crf in loop:
                        crf.pop_frame()
                mark()
            else:
                group.push_label_frames(labels, clusters)
                mark()
                group.set_proba(proba)
                group.reset_inferred()
                mark()
                group.inference(5)
                group.get_inferred(out=q_group)
                mark()
                if group.crfs[0].num_frames >= window:
                    group.pop_frame()
                mark()
            if i >= a.warmup:
                for k, x, y in zip(PARTS, t[:-1], t[1:]):
                    ms[mode][k].append((y - x) * 1e3)
                ms[mode]["step"].append((t[-1] - t[0]) * 1e3)
    same = [q_loop[b].cpu().numpy().tobytes() == q_group[b].cpu().numpy().tobytes() for b in range(B)]
    med = {mode: {k: float(np.median(v)) for k, v in parts.items()} for mode, parts in ms.items()}
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), card=card, frames=a.frames, streams=B,
                          slic_batch_ms=float(np.median(slic_ms)),
                          crf_ms_per_step_720p_K1600_C21_window3=med,
                          crf_step_speedup=med["loop"]["step"] / med["group"]["step"],
                          members_bit_identical=sum(same)), indent=1))
    if not all(same):
        sys.exit("members %s: the group's last q differs from the loop's" % [b for b, s in enumerate(same) if not s])


if __name__ == "__main__":
    main()
