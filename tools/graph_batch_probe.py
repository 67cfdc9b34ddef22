"""Cost of the batched label-map consumers at 1280x720, K=1600, batch 32 (DESIGN.md section 4.5).

Labels and clusters come from Slic.iterate_batch on the device.  Times, with CUDA events after warm-up, median of
--reps runs:
  (a) the three batched calls (get_connectivity_batch, get_mask_density_batch, broadcast_density_to_mask_batch) on
      cuda tensors, each alone and the three together;
  (b) the loop of 32 single-image host methods (SlicModel.get_connectivity / get_mask_density /
      broadcast_density_to_mask on numpy arrays): the route without the batch calls;
  (c) the per-image device entry points (fslic_b200_get_connectivity etc.) on device buffers, looped over 32 images.
Image 0 is checked against the compiled reference (oracle/_ref, where built) or its plain-C restatement.  Prints one
JSON line with the device name, power limit and maximum SM clock beside the numbers.

    python tools/graph_batch_probe.py [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fast_slic_b200 import CLUSTER_DTYPE, NodeConnectivity, Slic, SlicModel, _lib  # noqa: E402
from oracle.oracle import Port, Ref, synthetic_image  # noqa: E402


def _gpu_line():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def _event_ms(fn, reps):
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe needs a GPU"
    H, W, K, B = 720, 1280, 1600, 32
    s = Slic(num_components=K, min_size_factor=0.25)
    imgs = torch.from_numpy(np.stack([synthetic_image(H, W, seed=100 + b) for b in range(B)])).cuda()
    labels, clusters = s.iterate_batch(imgs, return_clusters=True)
    masks = torch.from_numpy(np.random.RandomState(7).randint(0, 256, (B, H, W)).astype(np.uint8)).cuda()
    dens = s.get_mask_density_batch(masks, labels, clusters)
    torch.cuda.synchronize()
    lab_np, mask_np = labels.cpu().numpy(), masks.cpu().numpy()
    cl_np = clusters.cpu().numpy().view(CLUSTER_DTYPE).reshape(B, K)

    def batched():
        s.get_connectivity_batch(labels)
        d = s.get_mask_density_batch(masks, labels, clusters)
        s.broadcast_density_to_mask_batch(d, labels)

    models = []
    for b in range(B):
        m = SlicModel(K)
        m._clusters = cl_np[b].copy()
        models.append(m)

    def host_loop():
        for b in range(B):
            m = models[b]
            m.get_connectivity(lab_np[b])
            d = m.get_mask_density(mask_np[b], lab_np[b])
            m.broadcast_density_to_mask(d, lab_np[b])

    L = _lib.lib()
    dev = labels.device
    nbytes = int(L.fslic_b200_connectivity_scratch_bytes(K))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    counts1 = torch.empty((B, K), dtype=torch.int32, device=dev)
    nb1 = torch.empty((B, K, 12), dtype=torch.int32, device=dev)
    dens1 = torch.empty((B, K), dtype=torch.uint8, device=dev)
    sum1 = torch.empty(K, dtype=torch.int32, device=dev)
    out1 = torch.empty((B, H, W), dtype=torch.uint8, device=dev)

    def device_loop():
        st = torch.cuda.current_stream(dev).cuda_stream
        for b in range(B):
            _lib.check(L.fslic_b200_get_connectivity(dev.index, H, W, K, labels[b].data_ptr(), counts1[b].data_ptr(),
                                                     nb1[b].data_ptr(), scratch.data_ptr(), nbytes, st))
            _lib.check(L.fslic_b200_get_mask_density(dev.index, H, W, K, clusters[b].data_ptr(), labels[b].data_ptr(),
                                                     masks[b].data_ptr(), dens1[b].data_ptr(), sum1.data_ptr(), st))
            _lib.check(L.fslic_b200_cluster_density_to_mask(dev.index, H, W, K, labels[b].data_ptr(), dens1[b].data_ptr(),
                                                            out1[b].data_ptr(), st))

    fns = {
        "batched_connectivity": lambda: s.get_connectivity_batch(labels),
        "batched_mask_density": lambda: s.get_mask_density_batch(masks, labels, clusters),
        "batched_broadcast": lambda: s.broadcast_density_to_mask_batch(dens, labels),
        "batched_all_three": batched,
        "host_single_image_loop": host_loop,
        "device_single_image_loop": device_loop,
    }
    for fn in fns.values():  # warm-up of every shape
        fn()
        fn()
    out = {"H": H, "W": W, "K": K, "batch": B, "reps": args.reps}
    for name, fn in fns.items():
        out[name + "_ms_median"] = _event_ms(fn, args.reps if not name.startswith("host") else max(3, args.reps // 3))

    # parity of image 0 (and the device loop's outputs against the batched ones)
    counts, nb = s.get_connectivity_batch(labels)
    d = s.get_mask_density_batch(masks, labels, clusters)
    bc = s.broadcast_density_to_mask_batch(d, labels)
    device_loop()
    torch.cuda.synchronize()
    checker = Ref() if Ref.available() else Port()
    lab0 = lab_np[0].view(np.uint16)
    ok = NodeConnectivity(counts[0].cpu().numpy(), nb[0].cpu().numpy()).tolist() == checker.get_connectivity(lab0, K)
    ok = ok and (d[0].cpu().numpy() == checker.get_mask_density(cl_np[0], lab0, mask_np[0])).all()
    ok = ok and (bc[0].cpu().numpy() == checker.density_to_mask(K, lab0, d[0].cpu().numpy())).all()
    out["checker"] = "reference" if isinstance(checker, Ref) else "port"
    out["image0_parity"] = bool(ok)
    out["device_loop_equals_batched"] = bool(torch.equal(counts, counts1) and torch.equal(nb, nb1) and
                                             torch.equal(d, dens1) and torch.equal(bc, out1))
    out["gpu"] = _gpu_line()
    print(json.dumps(out))
    if not (out["image0_parity"] and out["device_loop_equals_batched"]):
        sys.exit(1)


if __name__ == "__main__":
    main()
