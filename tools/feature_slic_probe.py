"""feature_slic at the 720p workload: 32 images of 1280x720, K = 1600, C in {3, 16, 64}, features resident in HBM.

Prints, as JSON lines (and, with --out FILE, writes the whole report there as JSON):
  * the card's name and power limit, read in the same run;
  * per C: the call's time (CUDA events, after warm-up, median of --reps), the per-kernel times of one call from
    torch.profiler (a separate run), the assign kernel's bytes (about 4 * C + 2 per visited pixel) over its time
    against 3.35 TB/s, the tiles that overflowed to the per-pixel kernel, and image 0 checked bit for bit against the
    numpy restatement (tests/feature_slic_cases.py);
  * as context, iterate_batch on uint8 RGB of the same size and K.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def features(B, C, H, W, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.arange(H, device="cuda", dtype=torch.float32)[:, None]
    x = torch.arange(W, device="cuda", dtype=torch.float32)[None, :]
    a = torch.rand((B, C, 3), generator=g, device="cuda") * 0.05 + 0.005
    f = torch.sin(x * a[..., 0, None, None] + y * a[..., 1, None, None] + a[..., 2, None, None] * 100) * 3
    return (f + torch.randn((B, C, H, W), generator=g, device="cuda") * 0.3).contiguous()


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms), min(ms), max(ms)


def kernel_times(fn):
    """{kernel name: [ms of each launch, in order]} of one call."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start):
        name = e.name.split("(")[0].replace("void ", "").split("<")[0].split("::")[-1]
        out.setdefault(name, []).append(e.time_range.elapsed_us() / 1000.0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--K", type=int, default=1600)
    ap.add_argument("--channels", default="3,16,64")
    ap.add_argument("--compactness", type=float, default=10.0)
    ap.add_argument("--max-iter", type=int, default=10)
    ap.add_argument("--stride", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-check", action="store_true")
    ap.add_argument("--out", default=None, help="also write the whole report to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("feature_slic_probe needs a CUDA device")
    from fast_slic_b200 import Slic
    from fast_slic_b200.feature_slic import feature_slic_dispatch, feature_slic
    B, H, W, K = a.batch, a.height, a.width, a.K
    report = {"card": card(), "workload": dict(B=B, H=H, W=W, K=K, compactness=a.compactness, max_iter=a.max_iter,
                                                stride=a.stride)}
    print(json.dumps(report["card"]), flush=True)
    rows = []
    for C in [int(c) for c in a.channels.split(",")]:
        x = features(B, C, H, W, seed=C)
        run = lambda: feature_slic(x, K, a.compactness, a.max_iter, a.stride)  # noqa: E731
        med, lo, hi = timed(run, a.reps, a.warmup)
        kt = kernel_times(run)
        tiles = kt.get("k_float_slic_assign_tiles", [])
        # the passes' visited pixels: max_iter strided passes, then the full one
        visited = [B * len(range(t % a.stride, H, a.stride)) * W for t in range(a.max_iter)] + [B * H * W]
        assign_bytes = [v * (4 * C + 2) for v in visited]
        full_ms = tiles[-1] if len(tiles) == len(visited) else None
        r, disp = feature_slic_dispatch(x, K, a.compactness, a.max_iter, a.stride)
        row = {"C": C, "call_ms_median": med, "call_ms_min": lo, "call_ms_max": hi,
               "kernels_ms": {k: round(sum(v), 4) for k, v in sorted(kt.items(), key=lambda kv: -sum(kv[1]))},
               "launches": {k: len(v) for k, v in kt.items()},
               "assign_ms_per_pass": [round(v, 4) for v in tiles],
               "full_assign_ms": full_ms,
               "full_assign_bytes": assign_bytes[-1],
               "full_assign_TBps": assign_bytes[-1] / full_ms / 1e9 if full_ms else None,
               "full_assign_share_of_3.35TBps": assign_bytes[-1] / full_ms / 1e9 / 3.35 if full_ms else None,
               "all_assign_bytes_over_assign_time_TBps": sum(assign_bytes) / sum(tiles) / 1e9 if tiles else None,
               "overflowed_tiles": [o for _, o in disp], "tiles": [t for t, _ in disp]}
        if not a.no_check:
            from feature_slic_cases import nan_class_equal, ref_feature_slic
            f0 = x[:1].cpu().numpy()
            final, pre, pos, mu, cnt = ref_feature_slic(f0, K, a.compactness, a.max_iter, a.stride)
            row["image0_exact"] = bool(np.array_equal(r.labels[:1].cpu().numpy(), final) and
                                       np.array_equal(r.count[:1].cpu().numpy(), cnt) and
                                       nan_class_equal(r.position[:1].cpu().numpy(), pos) and
                                       nan_class_equal(r.features[:1].cpu().numpy(), mu))
        print(json.dumps(row), flush=True)
        rows.append(row)
        del x
    report["feature_slic"] = rows
    imgs = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device="cuda")
    slic = Slic(num_components=K, compactness=10.0)
    med, lo, hi = timed(lambda: slic.iterate_batch(imgs, max_iter=a.max_iter), a.reps, a.warmup)
    report["iterate_batch_uint8_rgb"] = {"call_ms_median": med, "call_ms_min": lo, "call_ms_max": hi}
    print(json.dumps({"iterate_batch_uint8_rgb": report["iterate_batch_uint8_rgb"]}), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
