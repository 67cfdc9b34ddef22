"""Cost of superpixel merging at 1280x720, K=1600, batch 32 (DESIGN.md section 4.16).

Labels come from Slic.iterate_batch on the device; the region adjacency graph and the pooled-colour L2 weights are
built once, outside every timed window.  Times, with CUDA events after warm-up, median of --reps runs, of merge_regions
with a threshold (the median weight) and with num_regions=200, and of the route a user has without it: copy labels,
edges and weights to the host, then scipy's connected_components (threshold) or the Kruskal restatement of
tests/merge_cases.py (num_regions), then a numpy paint.  The host route is timed with a host clock, copies included.
Both routes' outputs must be equal before any time is printed.  With --profile, one torch.profiler pass adds the device
time of each kernel by name (take it in a run of its own: tracing slows the host).  Prints one JSON line with the
device name, power limit and maximum SM clock beside the numbers.

    python tools/merge_probe.py [--reps 20] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from fast_slic_b200 import Slic  # noqa: E402
from fast_slic_b200.merging import merge_regions  # noqa: E402
from fast_slic_b200.pooling import pool  # noqa: E402
from fast_slic_b200.region_graph import region_adjacency  # noqa: E402
from merge_cases import ref_merge, ref_paint, ref_present  # noqa: E402

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


def _host_ms(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


def _images(B, H, W, seed=5):
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[:H, :W].astype(np.float32)
    out = np.empty((B, H, W, 3), np.uint8)
    for b in range(B):
        f = rng.rand(3, 3) * 0.05
        base = 127 + 60 * np.sin(f[0, 0] * yy + f[0, 1] * xx)[..., None] * rng.rand(3)
        out[b] = np.clip(base + rng.randn(H, W, 3) * 8, 0, 255).astype(np.uint8)
    return torch.from_numpy(out).cuda()


def _host_threshold(labels, K, edge_index, weights, t):
    """Copy to the host, scipy connected components over the edges with weight < t, number by smallest member, paint."""
    lab = labels.cpu().numpy()
    src, dst = edge_index.cpu().numpy()
    w = weights.cpu().numpy()
    B = lab.shape[0]
    n = B * K
    present = ref_present(lab, K).reshape(-1)
    sel = (src < dst) & (w.astype(np.float64) < t)
    A = coo_matrix((np.ones(int(sel.sum()), np.int8), (src[sel], dst[sel])), shape=(n, n))
    _, comp = connected_components(A, directed=False)
    idx = np.arange(n)
    smallest = np.full(comp.max() + 1, n)
    np.minimum.at(smallest, comp[present], idx[present])
    root = smallest[comp]
    is_root = present & (root == idx)
    pos = np.cumsum(is_root) - is_root
    region = np.where(present, pos[np.minimum(root, n - 1)] - pos[idx // K * K], -1).astype(np.int32).reshape(B, K)
    return ref_paint(lab, region), region, is_root.reshape(B, K).sum(1).astype(np.int32)


def _host_count(labels, K, edge_index, weights, R):
    src, dst = edge_index.cpu().numpy()
    return ref_merge(labels.cpu().numpy(), K, src, dst, weights.cpu().numpy(), num_regions=R)


def _profile(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            fn()
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
    H, W, K, B, R = 720, 1280, 1600, 32, 200
    images = _images(B, H, W)
    labels = Slic(num_components=K, min_size_factor=0.25).iterate_batch(images)
    g = region_adjacency(labels, K)
    x = pool(images.permute(0, 3, 1, 2).float().contiguous(), labels, K).transpose(1, 2).reshape(-1, 3)
    w = (x[g.edge_index[0]] - x[g.edge_index[1]]).norm(dim=1)
    t = float(w.median())
    torch.cuda.synchronize()
    cuts = {"threshold": ({"threshold": t}, lambda: _host_threshold(labels, K, g.edge_index, w, t)),
            "num_regions": ({"num_regions": R}, lambda: _host_count(labels, K, g.edge_index, w, R))}
    for name, (kw, host) in cuts.items():
        ours = merge_regions(labels, K, g, w, **kw)
        theirs = host()
        for f, a, b in zip(ours._fields, ours, theirs):
            assert np.array_equal(a.cpu().numpy(), b), "%s: %s differs from the host route" % (name, f)
    if args.profile:
        res = {"gpu": _gpu_line(), "profile_ms": {name: _profile(lambda kw=kw: merge_regions(labels, K, g, w, **kw))
                                                  for name, (kw, _) in cuts.items()}}
        print(json.dumps(res))
        return
    n = B * H * W
    res = {"gpu": _gpu_line(), "H": H, "W": W, "K": K, "B": B, "reps": args.reps, "threshold": t, "num_regions": R,
           "directed_edges": int(g.edge_index.shape[1]), "equal_to_host": True,
           "ms": {"merge_" + name: round(_event_ms(lambda kw=kw: merge_regions(labels, K, g, w, **kw), args.reps), 4)
                  for name, (kw, _) in cuts.items()},
           # the paint's least traffic, labels in and regions out, over the data-sheet bandwidth
           "paint_min_bytes_ms": round(4 * n / HBM_BYTES_PER_MS, 4)}
    res["ms"].update({"host_" + name: round(_host_ms(host, max(3, args.reps // 4)), 2)
                      for name, (_, host) in cuts.items()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
