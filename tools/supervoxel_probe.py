"""supervoxel_slic on volume workloads, volumes resident in HBM:
  ct     4 volumes of 256 x 512 x 512 (D x H x W), C = 1, K = 16384 (CT-like)
  mri    8 volumes of 155 x 240 x 240, C = 4, K = 4000 (multi-modal MRI-like)
  aniso  2 volumes of 64 x 512 x 512, C = 1, K = 8192, spacing (3.0, 0.7, 0.7)

Prints, as JSON lines (and, with --out FILE, writes the whole report there as JSON):
  * the card's name and power limit, read in the same run;
  * per workload: the call's time (CUDA events, after warm-up, median of --reps); the per-kernel times of one call
    from torch.profiler (a separate run); the bytes of the full assign pass (4 * C + 2 per voxel) over its kernel time
    against 3.35 TB/s; the enforcement kernels' share of the call's kernel time; the peak memory of the call; the tiles
    that overflowed to the per-voxel kernel; and, for the workloads named by --check, volume 0 checked bit for bit
    against the numpy restatement (tests/supervoxel_cases.py; minutes of CPU time per workload).
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

WORKLOADS = {
    "ct": dict(B=4, C=1, D=256, H=512, W=512, K=16384, spacing=(1.0, 1.0, 1.0)),
    "mri": dict(B=8, C=4, D=155, H=240, W=240, K=4000, spacing=(1.0, 1.0, 1.0)),
    "aniso": dict(B=2, C=1, D=64, H=512, W=512, K=8192, spacing=(3.0, 0.7, 0.7)),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def volumes(B, C, D, H, W, seed=0):
    """Smooth float32 volumes with noise, made on the device volume by volume."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((B, C, D, H, W), dtype=torch.float32, device="cuda")
    z = torch.arange(D, device="cuda", dtype=torch.float32)[:, None, None]
    y = torch.arange(H, device="cuda", dtype=torch.float32)[None, :, None]
    x = torch.arange(W, device="cuda", dtype=torch.float32)[None, None, :]
    for b in range(B):
        for c in range(C):
            a = torch.rand(4, generator=g, device="cuda") * 0.05 + 0.005
            out[b, c] = torch.sin(x * a[0] + y * a[1] + z * a[2] + a[3] * 100) * 3
            out[b, c] += torch.randn((D, H, W), generator=g, device="cuda") * 0.3
    return out


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
    ap.add_argument("--workloads", default="ct,mri,aniso")
    ap.add_argument("--compactness", type=float, default=10.0)
    ap.add_argument("--max-iter", type=int, default=10)
    ap.add_argument("--stride", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check", default="", help="workloads whose volume 0 is checked against the restatement")
    ap.add_argument("--out", default=None, help="also write the whole report to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("supervoxel_probe needs a CUDA device")
    from fast_slic_b200.supervoxels import supervoxel_dispatch, supervoxel_slic
    check = set(filter(None, a.check.split(",")))
    report = {"card": card(), "settings": dict(compactness=a.compactness, max_iter=a.max_iter, stride=a.stride)}
    print(json.dumps(report["card"]), flush=True)
    rows = []
    for name in a.workloads.split(","):
        w = WORKLOADS[name]
        B, C, D, H, W, K, sp = w["B"], w["C"], w["D"], w["H"], w["W"], w["K"], w["spacing"]
        x = volumes(B, C, D, H, W, seed=len(rows))
        run = lambda: supervoxel_slic(x, K, a.compactness, sp, a.max_iter, a.stride)  # noqa: E731
        run()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        run()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        med, lo, hi = timed(run, a.reps, a.warmup)
        kt = kernel_times(run)
        total = sum(sum(v) for v in kt.values())
        enforce = sum(sum(v) for k, v in kt.items() if k.startswith("k_svc"))
        tiles = kt.get("k_float_slic_assign_tiles", [])
        fallback = kt.get("k_float_slic_assign_fallback", [])
        n = B * D * H * W
        full_bytes = n * (4 * C + 2)
        chunks = len(tiles) // (a.max_iter + 1) if tiles else 0
        # the full pass of each chunk is its last assign pass; the assign time of a pass is tile + fallback kernel
        full_ms = None
        if chunks and len(fallback) == len(tiles):
            per = a.max_iter + 1
            full_ms = sum(tiles[(c + 1) * per - 1] + fallback[(c + 1) * per - 1] for c in range(chunks))
        r, disp = supervoxel_dispatch(x, K, a.compactness, sp, a.max_iter, a.stride)
        row = {"workload": name, **{k: v for k, v in w.items()}, "grid": list(r.grid),
               "call_ms_median": med, "call_ms_min": lo, "call_ms_max": hi,
               "peak_bytes_beyond_inputs": int(peak),
               "kernels_ms": {k: round(sum(v), 4) for k, v in sorted(kt.items(), key=lambda kv: -sum(kv[1]))},
               "launches": {k: len(v) for k, v in kt.items()},
               "kernel_ms_total": total,
               "enforcement_ms": enforce, "enforcement_share_of_kernel_time": enforce / total if total else None,
               "full_assign_ms": full_ms, "full_assign_bytes": full_bytes,
               "full_assign_TBps": full_bytes / full_ms / 1e9 if full_ms else None,
               "full_assign_share_of_3.35TBps": full_bytes / full_ms / 1e9 / 3.35 if full_ms else None,
               "overflowed_tiles": [o for _, o in disp], "tiles": [t for t, _ in disp]}
        if name in check:
            from supervoxel_cases import nan_class_equal, ref_supervoxel_slic
            f0 = x[:1].cpu().numpy()
            final, pre, pos, mu, cnt, grid = ref_supervoxel_slic(f0, K, a.compactness, sp, a.max_iter, a.stride)
            row["volume0_exact"] = bool(np.array_equal(r.labels[:1].cpu().numpy(), final) and
                                        np.array_equal(r.count[:1].cpu().numpy(), cnt) and
                                        nan_class_equal(r.position[:1].cpu().numpy(), pos) and
                                        nan_class_equal(r.features[:1].cpu().numpy(), mu))
        else:
            row["volume0_exact"] = "not checked"
        print(json.dumps(row), flush=True)
        rows.append(row)
        del x, r
        torch.cuda.empty_cache()
    report["supervoxel_slic"] = rows
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
