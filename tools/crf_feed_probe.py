"""Times the SimpleCRF video loop fed through the host against the same loop fed from device tensors.

Both runs play the same frames: warm-started Slic.iterate_batch on the GPU at 1280x720 with K = 1600, then C = 21
class probabilities per superpixel, inference(5) over a sliding window of 3 frames, the newest frame's q read back, and
pop_frame.  They differ in how the CRF is fed:

  host    labels and records downloaded, push_slic_frame, set_proba(numpy), get_inferred() -> numpy
  device  push_label_frames(tensors), set_proba(cuda tensor), get_inferred(out=cuda tensor)

Each part is followed by a device synchronisation, so its wall time includes the GPU work it enqueued.  Reports the
median per frame and per part, and checks that the last frame's q of both runs is bit-identical.

    python tools/crf_feed_probe.py [--frames 40]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(mode, frames, K=1600, Cc=21, window=3, warmup=5):
    import torch
    from fast_slic_b200 import Slic, SlicModel
    from fast_slic_b200.crf import SimpleCRF
    from oracle.oracle import synthetic_image
    imgs = [torch.from_numpy(synthetic_image(720, 1280, seed=s)[None]).cuda() for s in range(4)]
    rng = np.random.RandomState(0)
    probas = [rng.dirichlet(np.ones(Cc), K).T.astype(np.float32).copy() for _ in range(8)]
    d_probas = [torch.from_numpy(p).cuda() for p in probas]
    slic = Slic(num_components=K)
    crf = SimpleCRF(Cc, K)
    model = SlicModel(K)
    q_dev = torch.empty(Cc, K, device="cuda")
    names = ("slic", "download", "push", "set_proba", "inference5_get", "pop")
    parts = {k: [] for k in names + ("frame",)}
    clusters = None
    q = None
    for i in range(frames + warmup):
        t = [time.perf_counter()]

        def mark():
            torch.cuda.synchronize()
            t.append(time.perf_counter())

        labels, clusters = slic.iterate_batch(imgs[i % 4], clusters=clusters, return_clusters=True)
        mark()
        if mode == "host":
            lab = labels[0].cpu().numpy()
            model._clusters = clusters[0].cpu().numpy().view(model._clusters.dtype).reshape(-1)
            mark()
            f = crf.push_slic_frame(types.SimpleNamespace(slic_model=model, last_assignment=lab))
            mark()
            f.set_proba(probas[i % 8])
            f.reset_inferred()
            mark()
            crf.inference(5)
            q = f.get_inferred()
            mark()
        else:
            mark()
            f = crf.push_label_frames(labels[0], clusters[0])
            mark()
            f.set_proba(d_probas[i % 8])
            f.reset_inferred()
            mark()
            crf.inference(5)
            f.get_inferred(out=q_dev)
            mark()
        if crf.num_frames >= window:
            crf.pop_frame()
        mark()
        if i >= warmup:
            for k, a, b in zip(names, t[:-1], t[1:]):
                parts[k].append((b - a) * 1e3)
            parts["frame"].append((t[-1] - t[0]) * 1e3)
    if mode == "device":
        q = q_dev.cpu().numpy()
    return {k: float(np.median(v)) for k, v in parts.items()}, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    a = ap.parse_args()
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    host_ms, q_host = run("host", a.frames)
    dev_ms, q_dev = run("device", a.frames)
    same = q_host.tobytes() == q_dev.tobytes()
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), card=card, frames=a.frames,
                          video_720p_K1600_C21_window3_ms_per_frame=dict(host_fed=host_ms, device_fed=dev_ms),
                          last_q_bit_identical=same), indent=1))
    if not same:
        sys.exit("the device-fed run's last q differs from the host-fed run's")


if __name__ == "__main__":
    main()
