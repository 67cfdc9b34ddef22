"""Cost of scoring superpixels against ground truth at 1280x720, K=1600, batch 32 (DESIGN.md section 4.14).

Images are 24x24-pixel patches of 21 classes, each class its own colour, so the class map is the ground truth and its
boundaries follow image edges; labels come from Slic.iterate_batch on the device.  Times, with CUDA events after
warm-up, median of --reps runs, of class_histogram (C = 21), segmentation_scores (tolerance 2) and boundaries, and of
what a user writes in torch without them: bincount over combined (image, label, class) keys for the histogram;
torch.unique(return_counts=True) over (image, label, gt) keys plus scatter_reduce for ASA and UE; the boundary maps
by slicing, max_pool2d dilation and sums for the boundary terms.  Every output of the two routes is compared, and must
be equal, before any time is printed.  With --profile, one torch.profiler pass adds the device time of each kernel by
name (take it in a run of its own: tracing slows the host).  Prints one JSON line with the device name, power limit
and maximum SM clock beside the numbers.

    python tools/gt_probe.py [--reps 20] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fast_slic_b200 import Slic  # noqa: E402
from fast_slic_b200.groundtruth import boundaries, class_histogram, segmentation_scores  # noqa: E402

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


def _workload(B, H, W, C, seed=5):
    rng = np.random.RandomState(seed)
    palette = rng.randint(0, 256, (C, 3)).astype(np.uint8)
    small = rng.randint(0, C, (B, H // 24 + 1, W // 24 + 1))
    gt = np.ascontiguousarray(np.kron(small, np.ones((1, 24, 24), np.int64))[:, :H, :W]).astype(np.uint8)
    return torch.from_numpy(palette[gt]).cuda(), torch.from_numpy(gt).cuda()


def _torch_histogram(classes, labels, K, C):
    B = labels.shape[0]
    lab = labels.long() & 0xFFFF
    cls = classes.long()
    ok = (lab < K) & (cls >= 0) & (cls < C)
    key = ((torch.arange(B, device=labels.device).view(B, 1, 1) * K + lab) * C + cls)[ok]
    return torch.bincount(key, minlength=B * K * C).to(torch.int32).view(B, K, C)


def _torch_scores(labels, gt, K, r):
    B = labels.shape[0]
    dev = labels.device
    lab = labels.long() & 0xFFFF
    g = gt.long()
    valid = (g >= 0) & (g <= 2 ** 31 - 1)
    counted = valid & (lab < K)
    node = torch.arange(B, device=dev).view(B, 1, 1) * K + lab
    uniq, cnt = torch.unique((node * 2 ** 31 + g)[counted], return_counts=True)
    nd = uniq >> 31
    n_k = torch.zeros(B * K, dtype=torch.int64, device=dev).scatter_reduce(0, nd, cnt, "sum")
    mx = torch.zeros(B * K, dtype=torch.int64, device=dev).scatter_reduce(0, nd, cnt, "amax")
    img = torch.div(nd, K, rounding_mode="floor")
    pixels = n_k.view(B, K).sum(1)
    asa = mx.view(B, K).sum(1)
    ue = torch.zeros(B, dtype=torch.int64, device=dev).scatter_reduce(0, img, torch.minimum(cnt, n_k[nd] - cnt), "sum")
    sp = torch.zeros_like(lab, dtype=torch.bool)
    sp[:, :, :-1] |= lab[:, :, :-1] != lab[:, :, 1:]
    sp[:, :-1, :] |= lab[:, :-1, :] != lab[:, 1:, :]
    gb = torch.zeros_like(sp)
    gb[:, :, :-1] |= valid[:, :, :-1] & valid[:, :, 1:] & (g[:, :, :-1] != g[:, :, 1:])
    gb[:, :-1, :] |= valid[:, :-1, :] & valid[:, 1:, :] & (g[:, :-1, :] != g[:, 1:, :])

    def dilate(m):
        return F.max_pool2d(m.float()[:, None], 2 * r + 1, stride=1, padding=r)[:, 0] > 0

    spv = sp & valid
    return torch.stack([pixels, asa, ue, gb.sum((1, 2)), (gb & dilate(sp)).sum((1, 2)), spv.sum((1, 2)),
                        (spv & dilate(gb)).sum((1, 2))])


def _torch_boundaries(labels):
    sp = torch.zeros_like(labels, dtype=torch.bool)
    sp[:, :, :-1] |= labels[:, :, :-1] != labels[:, :, 1:]
    sp[:, :-1, :] |= labels[:, :-1, :] != labels[:, 1:, :]
    return sp


def _profile(fns):
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for name, fn in fns.items():
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
        out[name] = dict(sorted(table.items(), key=lambda kv: -kv[1]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe needs a GPU"
    H, W, K, B, C, r = 720, 1280, 1600, 32, 21, 2
    imgs, gt = _workload(B, H, W, C)
    labels = Slic(num_components=K, min_size_factor=0.25).iterate_batch(imgs)
    torch.cuda.synchronize()
    ours = {"class_histogram": lambda: class_histogram(gt, labels, K, C),
            "segmentation_scores": lambda: segmentation_scores(labels, gt, K, r),
            "boundaries": lambda: boundaries(labels)}
    theirs = {"class_histogram": lambda: _torch_histogram(gt, labels, K, C),
              "segmentation_scores": lambda: _torch_scores(labels, gt, K, r),
              "boundaries": lambda: _torch_boundaries(labels)}
    s = segmentation_scores(labels, gt, K, r)
    equal = {"class_histogram": bool(torch.equal(ours["class_histogram"](), theirs["class_histogram"]())),
             "segmentation_scores": bool(torch.equal(torch.stack(list(s[:7])), theirs["segmentation_scores"]())),
             "boundaries": bool(torch.equal(ours["boundaries"](), theirs["boundaries"]()))}
    assert all(equal.values()), "outputs differ from the torch route: %s" % equal
    res = {"gpu": _gpu_line(), "H": H, "W": W, "K": K, "B": B, "C": C, "tolerance": r, "reps": args.reps,
           "equal_to_torch": equal, "ms": {},
           "asa_mean": round(float(s.asa.mean()), 4), "boundary_recall_mean": round(float(s.boundary_recall.mean()), 4)}
    for name in ours:
        res["ms"][name] = {"ours": round(_event_ms(ours[name], args.reps), 4),
                           "torch": round(_event_ms(theirs[name], args.reps), 4)}
    # the least each call must read (labels 2 + gt 1 bytes per pixel) and write, over the data-sheet bandwidth
    n = B * H * W
    res["min_bytes_ms"] = {"class_histogram": round(3 * n / HBM_BYTES_PER_MS, 4),
                           "segmentation_scores": round(3 * n / HBM_BYTES_PER_MS, 4),
                           "boundaries": round(3 * n / HBM_BYTES_PER_MS, 4)}
    if args.profile:
        res["profile_ms"] = _profile(ours)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
