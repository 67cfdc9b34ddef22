"""Cost of region adjacency graphs at 1280x720, K=1600, batch 32, connectivity 4 and 8 (DESIGN.md section 4.13).

Labels come from Slic.iterate_batch on the device.  Times, with CUDA events after warm-up, median of --reps runs, of
region_adjacency (count, the host read of the edge total, fill), and of what a user writes in torch without it: the
valid differing pixel pairs as (low node, high node) keys, torch.unique(return_counts=True), both directions, a sort
by (source, target) and the CSR offsets by bincount + cumsum.  The three outputs of the two are compared, and must be
equal, before anything is printed.  Bytes are the labels the count must read (2 per pixel) over the 3.35 TB/s HBM3
data-sheet bandwidth.  With --profile, one torch.profiler pass per connectivity adds the device time of each kernel by
name.  Prints one JSON line with the device name, power limit and maximum SM clock beside the numbers.

    python tools/rag_probe.py [--reps 20] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fast_slic_b200 import Slic  # noqa: E402
from fast_slic_b200.region_graph import region_adjacency  # noqa: E402
from oracle.oracle import synthetic_image  # noqa: E402

HBM_BYTES_PER_MS = 3.35e9


def _gpu_line():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def _event_ms(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def _torch_rag(labels, K, connectivity):
    B = labels.shape[0]
    n = B * K
    lab = labels.long() & 0xFFFF
    node = lab + torch.arange(B, device=labels.device).view(B, 1, 1) * K
    pairs = [((lab[:, :, :-1], node[:, :, :-1]), (lab[:, :, 1:], node[:, :, 1:])),
             ((lab[:, :-1, :], node[:, :-1, :]), (lab[:, 1:, :], node[:, 1:, :]))]
    if connectivity == 8:
        pairs += [((lab[:, :-1, :-1], node[:, :-1, :-1]), (lab[:, 1:, 1:], node[:, 1:, 1:])),
                  ((lab[:, :-1, 1:], node[:, :-1, 1:]), (lab[:, 1:, :-1], node[:, 1:, :-1]))]
    keys = []
    for (la, na), (lc, nc) in pairs:
        ok = (la < K) & (lc < K) & (la != lc)
        keys.append((torch.minimum(na, nc) * n + torch.maximum(na, nc))[ok])
    uniq, counts = torch.unique(torch.cat(keys), return_counts=True)
    lo, hi = uniq // n, uniq % n
    src, dst, w = torch.cat([lo, hi]), torch.cat([hi, lo]), torch.cat([counts, counts])
    order = torch.argsort(src * n + dst)
    src, dst, w = src[order], dst[order], w[order].to(torch.int32)
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=labels.device)
    indptr[1:] = torch.cumsum(torch.bincount(src, minlength=n), 0)
    return indptr, torch.stack([src, dst]), w


def _profile(labels, K, connectivity):
    from torch.profiler import ProfilerActivity, profile
    region_adjacency(labels, K, connectivity)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            region_adjacency(labels, K, connectivity)
        torch.cuda.synchronize()
    table = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            table[e.key[:80]] = round(t / 5 / 1000.0, 4)  # ms per call
    return dict(sorted(table.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe needs a GPU"
    H, W, K, B = 720, 1280, 1600, 32
    s = Slic(num_components=K, min_size_factor=0.25)
    imgs = torch.from_numpy(np.stack([synthetic_image(H, W, seed=100 + b) for b in range(B)])).cuda()
    labels = s.iterate_batch(imgs)
    torch.cuda.synchronize()
    res = {"gpu": _gpu_line(), "H": H, "W": W, "K": K, "B": B, "reps": args.reps, "by_connectivity": {}}
    for conn in (4, 8):
        g = region_adjacency(labels, K, conn)
        want = _torch_rag(labels, K, conn)
        same = [bool(torch.equal(a, b)) for a, b in zip(g, want)]
        assert all(same), "region_adjacency differs from the torch route: %s" % same
        t = {"region_adjacency": _event_ms(lambda: region_adjacency(labels, K, conn), args.reps),
             "torch_unique_route": _event_ms(lambda: _torch_rag(labels, K, conn), args.reps)}
        r = {"ms": {k: round(v, 4) for k, v in t.items()}, "edges": int(g.boundary.numel()),
             "equal_to_torch": True, "label_bytes_hbm_fraction": round(2 * B * H * W / HBM_BYTES_PER_MS /
                                                                       t["region_adjacency"], 4)}
        if args.profile:
            r["profile_ms"] = _profile(labels, K, conn)
        res["by_connectivity"][conn] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
