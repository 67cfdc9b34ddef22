"""Times message passing (fast_slic_b200.message_passing) on the README's workload against torch's building blocks.

Workload: 32 SLIC maps of 1280x720 at K = 1600 (iterate_batch), their region adjacency graph (connectivity 4) and a
symmetric 8-NN graph over pooled RGB means and normalised centroids, node features [B*K, C] for C in 16, 64, 256.
For each graph and C, the forward and the forward + backward of
  edge_gather (target), edge_softmax (H = 4), aggregate sum (weight [E]), mean and max,
and as baselines the same sums with torch.sparse_csr_tensor @ x and with index_select + index_add_ / scatter_reduce,
in torch's default mode and under torch.use_deterministic_algorithms(True).  Times are CUDA events around 20 calls
after 5 warm-up calls (median of 5 windows), so they include launch gaps; the kernel times of our functions come from
a torch.profiler run of its own.  The HBM bound is the least traffic each call needs (every input read once, every
output written once) over 3.35 TB/s (H100 SXM data sheet).  The card's name and power limit are read in the same run.

    python tools/message_passing_probe.py [--out FILE] [--quick]

Prints a table; with --out FILE it also writes the whole report there as JSON.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM = 3.35e12


def timed(fn, reps=20, windows=5, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / reps)
    return float(np.median(ms))


def kernel_ms(fn, reps=20):
    """Summed device time of the kernels fn launches, per call (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    total = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        if ev.key.startswith(("k_mp", "void k_mp")):
            total += t
    return total / 1000.0 / reps


def workload(quick):
    from cases import make_image
    from fast_slic_b200 import Slic
    from fast_slic_b200.geometry import region_properties
    from fast_slic_b200.pooling import pool
    from fast_slic_b200.region_graph import knn_graph, region_adjacency
    B, H, W = (4, 360, 640) if quick else (32, 720, 1280)
    imgs = torch.from_numpy(np.stack([make_image("syn", H, W, seed=70 + b) for b in range(B)])).cuda()
    labels, clusters = Slic(num_components=1600).iterate_batch(imgs, return_clusters=True)
    K = int(clusters.shape[1])
    p = region_properties(labels, K)
    hw = torch.tensor([H, W], dtype=torch.float64, device="cuda")
    pts = torch.cat([pool(imgs.permute(0, 3, 1, 2).float().contiguous() / 255, labels, K).transpose(1, 2),
                     (p.centroid / hw).float()], -1).contiguous()
    return B, K, {"rag": region_adjacency(labels, K, 4), "knn8_sym": knn_graph(pts, 8, p.area > 0, symmetric=True)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="also write the report to this file as JSON")
    ap.add_argument("--quick", action="store_true", help="4 images of 640x360 (a rehearsal)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("message_passing_probe needs a CUDA device")
    from fast_slic_b200.message_passing import aggregate, edge_gather, edge_softmax
    card = {"name": torch.cuda.get_device_name(0)}
    try:
        card["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        card["power_limit"] = "not read: %s" % e
    B, K, graphs = workload(args.quick)
    rows = []
    for gname, g in graphs.items():
        N, E = B * K, int(g.edge_index.shape[1])
        row, col = torch.repeat_interleave(torch.arange(N, device="cuda"), g.indptr.diff()), g.edge_index[1]
        for C in (16, 64, 256):
            gen = torch.Generator(device="cuda").manual_seed(C)
            x = torch.randn(N, C, device="cuda", generator=gen).requires_grad_(True)
            w = torch.rand(E, device="cuda", generator=gen).requires_grad_(True)
            s = torch.randn(E, 4, device="cuda", generator=gen).requires_grad_(True)
            gN, gE, gS = torch.randn(N, C, device="cuda"), torch.randn(E, C, device="cuda"), torch.randn(E, 4, device="cuda")
            node, ent, idx = 4 * N * C, 4 * E * C, 8 * (N + 1) + 8 * E
            ours = {
                "edge_gather": (lambda: edge_gather(x, g), gE, idx + node + ent),
                "edge_softmax": (lambda: edge_softmax(s, g), gS, idx + 2 * 16 * E),
                "aggregate_sum_w": (lambda: aggregate(x, g, w), gN, idx + 4 * E + 2 * node),
                "aggregate_mean": (lambda: aggregate(x, g, reduce="mean"), gN, idx + 2 * node + 4 * N),
                "aggregate_max": (lambda: aggregate(x, g, reduce="max"), gN, idx + 3 * node),
            }
            A = torch.sparse_csr_tensor(g.indptr, col, w.detach(), (N, N))
            deg = g.indptr.diff().clamp_min(1).float()[:, None]

            def ia_sum():
                return torch.zeros(N, C, device="cuda").index_add_(0, row, x.index_select(0, col) * w[:, None])

            def ia_mean():
                return torch.zeros(N, C, device="cuda").index_add_(0, row, x.index_select(0, col)) / deg

            def sr_max():
                return torch.zeros(N, C, device="cuda").scatter_reduce(0, row[:, None].expand(E, C),
                                                                       x.index_select(0, col), "amax",
                                                                       include_self=False)
            base = {"csr_matmul_sum_w": (lambda: A @ x, gN), "index_add_sum_w": (ia_sum, gN),
                    "index_add_mean": (ia_mean, gN), "scatter_reduce_max": (sr_max, gN)}
            for name, (fn, grad, nbytes) in ours.items():
                fwd = timed(lambda: fn())
                fb = timed(lambda: torch.autograd.backward(fn(), grad))
                kf = kernel_ms(lambda: fn())
                rows.append(dict(graph=gname, C=C, N=N, E=E, impl="ours", op=name, fwd_ms=fwd, fwd_bwd_ms=fb,
                                 fwd_kernel_ms=kf, hbm_bound_ms=nbytes / HBM * 1e3,
                                 fwd_kernel_hbm_share=nbytes / HBM * 1e3 / kf if kf else None))
            for det in (False, True):
                torch.use_deterministic_algorithms(det)
                for name, (fn, grad) in base.items():
                    r = dict(graph=gname, C=C, N=N, E=E, impl="torch_deterministic" if det else "torch_default", op=name)
                    for key, call in (("fwd_ms", lambda: fn()), ("fwd_bwd_ms", lambda: torch.autograd.backward(fn(), grad))):
                        try:
                            r[key] = timed(call)
                        except Exception as e:  # noqa: BLE001  (an op torch does not offer in this mode)
                            r[key] = "unsupported: %s" % str(e).splitlines()[0][:120]
                    rows.append(r)
                torch.use_deterministic_algorithms(False)
            x.grad = w.grad = s.grad = None
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card, "B": B, "K": K, "rows": rows}, f, indent=1)
    print(json.dumps(card))
    for r in rows:
        print("%-9s C=%-3d %-20s %-20s fwd %s  fwd+bwd %s  kernels %s  hbm %s" % (
            r["graph"], r["C"], r["impl"], r["op"], _f(r.get("fwd_ms")), _f(r.get("fwd_bwd_ms")),
            _f(r.get("fwd_kernel_ms")), _f(r.get("fwd_kernel_hbm_share"), "%.2f")))


def _f(v, fmt="%.4f"):
    return fmt % v if isinstance(v, float) else ("-" if v is None else str(v)[:40])


if __name__ == "__main__":
    main()
