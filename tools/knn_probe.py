"""Cost of knn_graph (DESIGN.md section 4.18) on two workloads:
- hd: README's node features of 32 1280x720 SLIC maps at K = 1600 (pooled RGB means, normalised centroids,
  compactness: D = 6), present = area > 0, k = 8, directed and symmetric;
- 4k: one 3840x2160 SLIC map at K = 65534, D = 5 (pooled RGB means and normalised centroids), k = 8, directed and
  symmetric.
Times, with CUDA events after warm-up, median of --reps runs, of knn_graph (host read included) and of what a user
writes in torch without it: torch.cdist(compute_mode="donot_use_mm_for_euclid_dist"), masking of absent nodes and
self loops, topk (over blocks of 1024 query rows when K is larger: torch.cdist cannot launch over 65534^2 distances
at once), and CSR assembly (for the symmetric graph, to_undirected's unique of both directions).  Where cdist's
[B,K,K] tables would not fit the free device memory, the torch route is marked not run.  Before timing, each row's
sorted distances are compared with the torch route's squared ones, within 1e-5 relative (torch's order among ties
is undefined, so edge lists are not compared); the probe fails when they differ.  With --profile, one torch.profiler pass per case adds the device time of
each kernel by name.  The FP32 floor of the select kernel is B * K^2 * 3D operations over the data sheet's 67 TFLOP/s.
Prints one JSON line with the device name, power limit and maximum SM clock beside the numbers.

    python tools/knn_probe.py [--reps 20] [--profile]
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
from fast_slic_b200.geometry import region_properties  # noqa: E402
from fast_slic_b200.pooling import pool  # noqa: E402
from fast_slic_b200.region_graph import knn_graph  # noqa: E402
from oracle.oracle import synthetic_image  # noqa: E402

FP32_TFLOPS = 67.0  # H100 SXM data sheet, dense FP32


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


def _points(H, W, K, B, seed, compactness):
    """README's node features of B SLIC maps, padded with absent rows to K nodes per image (Slic takes fewer than
    65534 components)."""
    imgs = torch.from_numpy(np.stack([synthetic_image(H, W, seed=seed + b) for b in range(B)])).cuda()
    labels, clusters = Slic(num_components=min(K, 65533)).iterate_batch(imgs, return_clusters=True)
    n = int(clusters.shape[1])
    p = region_properties(labels, n)
    hw = torch.tensor([H, W], dtype=torch.float64, device="cuda")
    parts = [pool(imgs.permute(0, 3, 1, 2).float().contiguous() / 255, labels, n).transpose(1, 2),
             (p.centroid / hw).float()]
    if compactness:
        parts.append((p.perimeter / p.area.clamp(min=1)).float()[..., None])
    x = torch.cat(parts, -1)
    pad = max(K, n) - n
    x = torch.cat([x, x.new_zeros(B, pad, x.shape[2])], 1).contiguous()
    present = torch.cat([p.area > 0, torch.zeros(B, pad, dtype=torch.bool, device="cuda")], 1)
    return x, present


def _torch_knn(x, k, present, symmetric, rows):
    B, K, _ = x.shape
    vals, idxs = [], []
    for r0 in range(0, K, rows):  # query rows in blocks: cdist cannot launch over 65534^2 at once
        d = torch.cdist(x[:, r0:r0 + rows], x, compute_mode="donot_use_mm_for_euclid_dist")
        d.masked_fill_(~present[:, None, :], float("inf"))
        d.diagonal(offset=r0, dim1=1, dim2=2).fill_(float("inf"))
        v, i = d.topk(k, dim=2, largest=False)
        vals.append(v)
        idxs.append(i)
        del d
    val, idx = torch.cat(vals, 1), torch.cat(idxs, 1)  # [B,K,k]
    keep = present[:, :, None] & torch.isfinite(val)
    src = (torch.arange(B * K, device=x.device).view(B, K, 1)).expand(B, K, k)[keep]
    dst = (idx + torch.arange(B, device=x.device).view(B, 1, 1) * K)[keep]
    dist = (val * val)[keep]
    N = B * K
    if symmetric:
        key, inverse = torch.unique(torch.cat([src * N + dst, dst * N + src]), return_inverse=True)
        w = torch.empty(key.numel(), device=x.device).scatter_(0, inverse, torch.cat([dist, dist]))
        src, dst, dist = key // N, key % N, w
    else:
        order = torch.argsort(src * N + dst)
        src, dst, dist = src[order], dst[order], dist[order]
    indptr = torch.zeros(N + 1, dtype=torch.int64, device=x.device)
    indptr[1:] = torch.cumsum(torch.bincount(src, minlength=N), 0)
    return indptr, torch.stack([src, dst]), dist


def _rows_agree(g, ref):
    """Same row lengths and each row's sorted distances within 1e-5 relative."""
    if not torch.equal(g.indptr, ref[0]):
        return False
    rows = torch.repeat_interleave(torch.arange(g.indptr.numel() - 1, device=g.indptr.device), g.indptr.diff())

    def row_sorted(d):
        o = torch.argsort(d, stable=True)
        return d[o[torch.argsort(rows[o], stable=True)]].double()

    a, b = row_sorted(g.distance), row_sorted(ref[2])
    return bool(((a - b).abs() <= 1e-5 * b.abs()).all())


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
    res = {"gpu": _gpu_line(), "reps": args.reps, "cases": {}}
    k = 8
    for name, (H, W, K, B, compactness) in (("hd", (720, 1280, 1600, 32, True)), ("4k", (2160, 3840, 65534, 1, False))):
        x, present = _points(H, W, K, B, 100, compactness)
        B, K, D = x.shape
        torch.cuda.synchronize()
        free = torch.cuda.mem_get_info()[0]
        rows = K if K <= 1024 else 1024
        fits = 3 * B * rows * K * 4 < free  # cdist's table, its topk and the mask
        flops = B * K * K * 3 * D
        for sym in (False, True):
            g = knn_graph(x, k, present, sym)
            r = {"B": B, "K": K, "D": D, "k": k, "symmetric": sym, "edges": int(g.edge_index.shape[1]),
                 "candidates": int(present.sum()), "torch_rows_per_block": rows, "select_fp32_ops": flops,
                 "fp32_floor_ms": round(flops / (FP32_TFLOPS * 1e12) * 1e3, 4)}
            t = {"knn_graph": _event_ms(lambda: knn_graph(x, k, present, sym), args.reps)}
            if fits:
                ref = _torch_knn(x, k, present, sym, rows)
                r["rows_agree_with_torch"] = _rows_agree(g, ref)
                del ref
                t["torch_route"] = _event_ms(lambda: _torch_knn(x, k, present, sym, rows), max(3, args.reps // 4))
            else:
                t["torch_route"] = "not run: cdist needs %.1f GB, %.1f GB free" % (3 * B * rows * K * 4 / 1e9, free / 1e9)
            r["ms"] = {n: (round(v, 4) if isinstance(v, float) else v) for n, v in t.items()}
            if args.profile:
                r["profile_ms"] = _profile(lambda: knn_graph(x, k, present, sym))
            res["cases"]["%s_%s" % (name, "symmetric" if sym else "directed")] = r
            torch.cuda.empty_cache()
    print(json.dumps(res))
    if not all(r.get("rows_agree_with_torch", True) for r in res["cases"].values()):
        sys.exit("knn_graph's rows differ from the torch route's")


if __name__ == "__main__":
    main()
