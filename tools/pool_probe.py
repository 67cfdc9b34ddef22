"""Cost of superpixel pooling at 1280x720, K=1600, batch 32, C in {1, 21, 64} (DESIGN.md section 4.12).

Labels come from Slic.iterate_batch on the device.  Times, with CUDA events after warm-up, median of --reps runs, of
  pool (mean, sort included), unpool, paint_argmax, and one autograd backward of the mean (unpool(grad) / count),
and, at the same sizes, what a user writes in torch without them: scatter_add_ over labels.long() into [B,C,K]
(float atomics) plus the counts and the division, torch.gather for unpool, argmax + gather for paint_argmax.  The
outputs of the two are compared (means within float tolerance, the gathers exactly).  Bytes are what each call has to
move, from the shapes: pool reads features and labels and writes [B,C,K] and the counts; unpool reads labels and
[B,C,K] and writes features; paint_argmax reads labels and q and writes int16 classes.  The fraction is of the
3.35 TB/s HBM3 data-sheet bandwidth.  With --profile, one torch.profiler pass over pool at C=21 adds the kernel times
by name.  Prints one JSON line with the device name, power limit and maximum SM clock beside the numbers.

    python tools/pool_probe.py [--reps 20] [--profile]
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
from fast_slic_b200.pooling import paint_argmax, pool, unpool  # noqa: E402
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


def _torch_pool(feats, labels, K):
    B, C = feats.shape[:2]
    lab = labels.long().view(B, 1, -1)  # the int64 copy
    valid = (lab >= 0) & (lab < K)
    idx = torch.where(valid, lab, K)  # one spare bin for labels outside [0, K)
    sums = torch.zeros((B, C, K + 1), dtype=torch.float32, device=feats.device)
    sums.scatter_add_(2, idx.expand(B, C, -1), feats.view(B, C, -1))
    counts = torch.zeros((B, K + 1), dtype=torch.float32, device=feats.device)
    counts.scatter_add_(1, idx[:, 0], valid[:, 0].float())
    return torch.where(counts[:, None, :K] > 0, sums[:, :, :K] / counts[:, None, :K], 0.0)


def _torch_unpool(values, labels):
    B, C, K = values.shape
    lab = labels.long().view(B, 1, -1)
    valid = (lab >= 0) & (lab < K)
    g = torch.gather(values, 2, torch.where(valid, lab, 0).expand(B, C, -1))
    return torch.where(valid, g, 0.0).view(B, C, *labels.shape[1:])


def _torch_paint(q, labels):
    B, C, K = q.shape
    lab = labels.long().view(B, -1)
    valid = (lab >= 0) & (lab < K)
    cls = torch.gather(torch.argmax(q, dim=1), 1, torch.where(valid, lab, 0))
    return torch.where(valid, cls, -1).to(torch.int16).view(labels.shape)


def _profile(feats, labels, K):
    from torch.profiler import ProfilerActivity, profile
    pool(feats, labels, K)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            pool(feats, labels, K)
        torch.cuda.synchronize()
    table = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            table[e.key[:80]] = round(t / 5 / 1000.0, 4)  # ms per pool call
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
    n = B * H * W
    res = {"gpu": _gpu_line(), "H": H, "W": W, "K": K, "B": B, "reps": args.reps, "by_C": {}}
    for C in (1, 21, 64):
        feats = torch.randn((B, C, H, W), device="cuda")
        q = torch.rand((B, C, K), device="cuda")
        grad = torch.randn((B, C, K), device="cuda")
        means = pool(feats, labels, K)
        err = float((means - _torch_pool(feats, labels, K)).abs().max())
        same_unpool = bool(torch.equal(unpool(q, labels), _torch_unpool(q, labels)))
        same_paint = bool(torch.equal(paint_argmax(q, labels), _torch_paint(q, labels)))
        f = feats.clone().requires_grad_()
        out = pool(f, labels, K)

        def backward():
            f.grad = None
            out.backward(grad, retain_graph=True)

        t = {"pool": _event_ms(lambda: pool(feats, labels, K), args.reps),
             "unpool": _event_ms(lambda: unpool(q, labels), args.reps),
             "paint_argmax": _event_ms(lambda: paint_argmax(q, labels), args.reps),
             "pool_backward": _event_ms(backward, args.reps),
             "torch_scatter_add_pool": _event_ms(lambda: _torch_pool(feats, labels, K), args.reps),
             "torch_gather_unpool": _event_ms(lambda: _torch_unpool(q, labels), args.reps),
             "torch_argmax_gather_paint": _event_ms(lambda: _torch_paint(q, labels), args.reps)}
        small = B * C * K * 4
        nbytes = {"pool": n * (4 * C + 2) + small + B * K * 4, "unpool": n * (4 * C + 2) + small,
                  "paint_argmax": n * 4 + small, "pool_backward": n * (4 * C + 2) + small + B * K * 4}
        res["by_C"][C] = {
            "ms": {k: round(v, 4) for k, v in t.items()},
            "GB": {k: round(v / 1e9, 3) for k, v in nbytes.items()},
            "hbm_fraction": {k: round(v / HBM_BYTES_PER_MS / t[k], 3) for k, v in nbytes.items()},
            "max_abs_diff_mean_vs_torch": err, "unpool_equal_torch": same_unpool, "paint_equal_torch": same_paint,
        }
        del feats, q, grad, f, out, means
    if args.profile:
        feats = torch.randn((B, 21, H, W), device="cuda")
        res["profile_pool_C21_ms"] = _profile(feats, labels, K)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
