"""Cost of boundary statistics at 1280x720, K=1600, batch 32, C in {1, 16}, connectivity 4 and 8 (DESIGN.md section
4.17).

Labels come from Slic.iterate_batch on the device, the graph from region_adjacency, the values from a seeded uniform
draw in [0, 1) (a boundary probability map).  Times, with CUDA events after warm-up, median of --reps runs, of boundary_stats (selection, the host read of the
pair count, keys, sorts, the run reduction), and of what a user writes in torch without it: the valid differing pixel
pairs as (low node, high node) keys, torch.unique(return_inverse=True, return_counts=True), index_add_ of the anchor
and other values (float atomics), scatter_reduce amin / amax, and searchsorted of the graph's entries.  count, min and
max must equal the torch route's and mean be within 1e-5 relative of it before anything is printed.  With --profile,
one torch.profiler pass per case adds the device time of each kernel by name.  Prints one JSON line with the device
name, power limit and maximum SM clock beside the numbers.

    python tools/boundary_probe.py [--reps 20] [--profile]
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
from fast_slic_b200.region_graph import boundary_stats, region_adjacency  # noqa: E402
from oracle.oracle import synthetic_image  # noqa: E402


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


def _torch_boundary(labels, K, graph, values, connectivity):
    B, C, H, W = values.shape
    n = B * K
    dev = labels.device
    lab = labels.long() & 0xFFFF
    node = lab + torch.arange(B, device=dev).view(B, 1, 1) * K
    pix = torch.arange(B * H * W, device=dev).view(B, H, W)
    sl = [((slice(None), slice(None), slice(None, -1)), (slice(None), slice(None), slice(1, None))),
          ((slice(None), slice(None, -1), slice(None)), (slice(None), slice(1, None), slice(None)))]
    if connectivity == 8:
        sl += [((slice(None), slice(None, -1), slice(None, -1)), (slice(None), slice(1, None), slice(1, None))),
               ((slice(None), slice(None, -1), slice(1, None)), (slice(None), slice(1, None), slice(None, -1)))]
    keys, pa, pc = [], [], []
    for a, c in sl:
        ok = (lab[a] < K) & (lab[c] < K) & (lab[a] != lab[c])
        keys.append((torch.minimum(node[a], node[c]) * n + torch.maximum(node[a], node[c]))[ok])
        pa.append(pix[a][ok])
        pc.append(pix[c][ok])
    uniq, inv, counts = torch.unique(torch.cat(keys), return_inverse=True, return_counts=True)
    pa, pc = torch.cat(pa), torch.cat(pc)
    v = values.permute(1, 0, 2, 3).reshape(C, -1)
    va, vc = v[:, pa], v[:, pc]
    U = uniq.numel()
    idx = inv.view(1, -1).expand(C, -1)
    sums = torch.zeros((C, U), device=dev).index_add_(1, inv, va).index_add_(1, inv, vc)
    mean = sums / (2 * counts).float()
    mn = torch.full((C, U), float("inf"), device=dev).scatter_reduce_(1, idx, va, "amin").scatter_reduce_(1, idx, vc,
                                                                                                          "amin")
    mx = torch.full((C, U), -float("inf"), device=dev).scatter_reduce_(1, idx, va, "amax").scatter_reduce_(1, idx, vc,
                                                                                                           "amax")
    src, dst = graph.edge_index
    ekey = torch.minimum(src, dst) * n + torch.maximum(src, dst)
    pos = torch.searchsorted(uniq, ekey).clamp_(max=max(U - 1, 0))
    found = (uniq[pos] == ekey) & (src != dst)
    nan = torch.tensor(float("nan"), device=dev)
    rows = [torch.where(found[:, None], t.t()[pos], nan) for t in (mean, mn, mx)]
    return rows[0], rows[1], rows[2], torch.where(found, counts[pos], 0).to(torch.int32)


def _profile(labels, K, g, values, connectivity):
    from torch.profiler import ProfilerActivity, profile
    boundary_stats(labels, K, g, values, connectivity)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            boundary_stats(labels, K, g, values, connectivity)
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
    gen = torch.Generator(device="cuda").manual_seed(5)
    res = {"gpu": _gpu_line(), "H": H, "W": W, "K": K, "B": B, "reps": args.reps, "cases": {}}
    for conn in (4, 8):
        g = region_adjacency(labels, K, conn)
        for C in (1, 16):
            values = torch.rand((B, C, H, W), device="cuda", generator=gen)  # a boundary probability map
            got = boundary_stats(labels, K, g, values, conn)
            want = _torch_boundary(labels, K, g, values, conn)
            assert torch.equal(got.count, want[3]) and torch.equal(got.count, g.boundary), "count differs"
            assert torch.equal(got.min, want[1]) and torch.equal(got.max, want[2]), "min / max differ"
            rel = ((got.mean.double() - want[0].double()).abs() / want[0].double().abs().clamp_min(1e-30)).max().item()
            assert rel <= 1e-5, "mean differs by %g relative" % rel
            t = {"boundary_stats": _event_ms(lambda: boundary_stats(labels, K, g, values, conn), args.reps),
                 "torch_route": _event_ms(lambda: _torch_boundary(labels, K, g, values, conn), args.reps)}
            r = {"ms": {k: round(v, 4) for k, v in t.items()}, "edges": int(g.boundary.numel()),
                 "boundary_pairs": int(g.boundary.long().sum().item()) // 2, "mean_max_rel_diff": rel}
            if args.profile:
                r["profile_ms"] = _profile(labels, K, g, values, conn)
            res["cases"]["conn%d_C%d" % (conn, C)] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
