"""Cost of superpixel shapes at 1280x720, K=1600, batch 32 (DESIGN.md section 4.15).

Labels come from Slic.iterate_batch on the device.  Times, with CUDA events after warm-up, median of --reps runs, of
region_properties and of what a user writes in torch without it: coordinate grids, scatter_add_ over labels.long() for
the area and moments, scatter_reduce("amin" / "amax") for the boxes, shifted-slice compares and another scatter_add_
for the perimeter and border, and the float fields by elementwise ops.  Every field of the two routes is compared, and
must be equal, before any time is printed.  With --profile, one torch.profiler pass adds the device time of each kernel
by name (take it in a run of its own: tracing slows the host).  Prints one JSON line with the device name, power limit
and maximum SM clock beside the numbers.

    python tools/geometry_probe.py [--reps 20] [--profile]
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

HBM_BYTES_PER_MS = 3.35e9
I32_MAX = 2 ** 31 - 1


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


def _images(B, H, W, seed=5):
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[:H, :W].astype(np.float32)
    out = np.empty((B, H, W, 3), np.uint8)
    for b in range(B):
        f = rng.rand(3, 3) * 0.05
        base = 127 + 60 * np.sin(f[0, 0] * yy + f[0, 1] * xx)[..., None] * rng.rand(3)
        out[b] = np.clip(base + rng.randn(H, W, 3) * 8, 0, 255).astype(np.uint8)
    return torch.from_numpy(out).cuda()


def _torch_route(labels, K):
    """The same fields with torch ops: [B,2,H,W] coordinates, scatters over the node index."""
    B, H, W = labels.shape
    dev = labels.device
    lab = labels.long() & 0xFFFF
    ok = lab < K
    node = torch.where(ok, torch.arange(B, device=dev).view(B, 1, 1) * K + lab, B * K).view(-1)  # B*K: a spill slot
    yx = torch.stack(torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij"))
    y, x = (c.expand(B, H, W).reshape(-1) for c in yx)
    N = B * K + 1
    mom = torch.stack([y, x, y * y, x * y, x * x], 1)
    area = torch.zeros(N, dtype=torch.int64, device=dev).scatter_add_(0, node, torch.ones_like(node))
    moments = torch.zeros((N, 5), dtype=torch.int64, device=dev).scatter_add_(0, node[:, None].expand(-1, 5), mom)
    lo = torch.stack([y, x], 1)
    bmin = torch.full((N, 2), I32_MAX, dtype=torch.int64, device=dev).scatter_reduce(
        0, node[:, None].expand(-1, 2), lo, "amin")
    bmax = torch.zeros((N, 2), dtype=torch.int64, device=dev).scatter_reduce(0, node[:, None].expand(-1, 2), lo + 1, "amax")
    # the sides of each pixel facing the image edge or another label
    pad = torch.full((B, H + 2, W + 2), -1, dtype=torch.int64, device=dev)
    pad[:, 1:-1, 1:-1] = lab
    sides = torch.zeros((B, H, W), dtype=torch.int64, device=dev)
    for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
        sides += pad[:, 1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx] != lab
    edge = torch.zeros((H, W), dtype=torch.int64, device=dev)
    edge[0] += 1
    edge[-1] += 1
    edge[:, 0] += 1
    edge[:, -1] += 1
    perimeter = torch.zeros(N, dtype=torch.int64, device=dev).scatter_add_(0, node, sides.view(-1))
    border = torch.zeros(N, dtype=torch.int64, device=dev).scatter_add_(0, node, edge.expand(B, H, W).reshape(-1))
    area, moments, perimeter, border = area[:-1], moments[:-1], perimeter[:-1], border[:-1]
    empty = area == 0
    bbox = torch.cat([bmin[:-1], bmax[:-1]], 1).masked_fill(empty[:, None], 0)
    n = area.double().clamp(min=1)
    q = moments.double() / n[:, None]
    cy, cx = q[:, 0], q[:, 1]
    cen = torch.stack([cy, cx], 1).masked_fill(empty[:, None], 0.0)
    cov = torch.stack([q[:, 2] - cy * cy, q[:, 3] - cy * cx, q[:, 4] - cx * cx], 1).masked_fill(empty[:, None], 0.0)
    return (area.int().view(B, K), bbox.int().view(B, K, 4), moments.view(B, K, 5), perimeter.int().view(B, K),
            border.int().view(B, K), cen.view(B, K, 2), cov.view(B, K, 3))


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
    H, W, K, B = 720, 1280, 1600, 32
    labels = Slic(num_components=K, min_size_factor=0.25).iterate_batch(_images(B, H, W))
    torch.cuda.synchronize()
    ours = region_properties(labels, K)
    theirs = _torch_route(labels, K)
    equal = {f: bool(torch.equal(a, b)) for f, a, b in zip(ours._fields, ours, theirs)}
    assert all(equal.values()), "outputs differ from the torch route: %s" % equal
    n = B * H * W
    runs = int(((labels[:, :, 1:] != labels[:, :, :-1]).sum() + B * H).item())
    res = {"gpu": _gpu_line(), "H": H, "W": W, "K": K, "B": B, "reps": args.reps, "equal_to_torch": equal,
           "mean_run_px": round(n / runs, 2), "nonempty": int((ours.area > 0).sum()),
           "ms": {"region_properties": round(_event_ms(lambda: region_properties(labels, K), args.reps), 4),
                  "torch": round(_event_ms(lambda: _torch_route(labels, K), args.reps), 4)},
           # the least traffic, the 2-byte labels, over the data-sheet bandwidth
           "min_bytes_ms": round(2 * n / HBM_BYTES_PER_MS, 4)}
    if args.profile:
        res["profile_ms"] = _profile(lambda: region_properties(labels, K))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
