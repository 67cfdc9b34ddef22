"""Per-kernel time of connectivity enforcement inside the bench workload.

python tools/cca_probe.py [--workload B] [--batch 32] [--steps 20] [--json OUT]

Runs Engine.iterate on seeded images from bench.synth_images_torch, one step after the other on one stream.  Two runs:
the step time from CUDA events with the profiler off, then the kernel times from torch.profiler (CUDA activities) in
a run of their own.  Kernels are grouped into the per-pixel front of the connectivity stage (k_ccl_tile, k_ccl_seams,
k_ccl_flatten), the std::partial_sort replay (k_cca_select) and the per-component back half (everything else of
cca.cuh).  Prints one table and, with --json, writes the same numbers to OUT."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FRONT = ("k_ccl_tile", "k_ccl_seams", "k_ccl_flatten")
SELECT = ("k_cca_select",)
BACK_PREFIXES = ("k_ccl_", "k_cca_", "k_kept_", "k_scan_blocks")


def kernel_name(full):
    """'void k_cca_absorb(CcaParams, ...)' -> 'k_cca_absorb' (template arguments dropped)."""
    head = full.split("(")[0].split("<")[0].strip()
    return head.split()[-1] if head else full


def group_of(name):
    if name in FRONT:
        return "front"
    if name in SELECT:
        return "select"
    if name.startswith(BACK_PREFIXES):
        return "back"
    return None


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        limit = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="B")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", metavar="OUT")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from bench import COMPACTNESS, MAX_ITER, STRIDE, WORKLOADS, synth_images_torch
    from fast_slic_b200 import get_engine

    if not torch.cuda.is_available():
        sys.exit("cca_probe needs a GPU")
    H, W, K, msf = WORKLOADS[args.workload]
    B = args.batch
    dev = torch.device("cuda", 0)
    npool = 4
    pool = synth_images_torch(npool * B, H, W, 1000, 12.0, dev).view(npool, B, H, W, 3)
    eng = get_engine(H, W, K, B, 0)
    pristine = eng.initialize_clusters(pool[0])
    clusters = pristine.clone()
    labels = torch.empty((B, H, W), dtype=torch.int16, device=dev)
    params = eng.params(COMPACTNESS, msf, STRIDE, True, MAX_ITER)

    def step(i):
        clusters.copy_(pristine)
        eng.iterate(pool[i % npool], clusters, params, labels)

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()

    # (1) step time, profiler off
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        step(i)
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / args.steps

    # (2) kernel times, a run of its own
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            step(i)
        torch.cuda.synchronize()
    per = {}
    total_us = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "self_device_time_total", None)
        if t is None:
            t = ev.self_cuda_time_total
        if t <= 0:
            continue
        us = t / args.steps
        total_us += us
        n = kernel_name(ev.key)
        if group_of(n):
            cnt = ev.count / args.steps
            prev = per.get(n, (0.0, 0.0))
            per[n] = (prev[0] + us, prev[1] + cnt)

    name, limit = card()
    groups = {"front": 0.0, "select": 0.0, "back": 0.0}
    rows = []
    for n, (us, cnt) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        g = group_of(n)
        groups[g] += us
        rows.append({"kernel": n, "group": g, "us_per_step": round(us, 1), "launches_per_step": cnt,
                     "share_of_kernel_time": round(us / total_us, 4), "share_of_step": round(us / (1e3 * step_ms), 4)})
    res = {"card": name, "power_limit_max_sm_clock": limit, "workload": args.workload, "H": H, "W": W, "K": K,
           "batch": B, "steps": args.steps, "step_ms": round(step_ms, 3), "kernel_us_per_step": round(total_us, 1),
           "groups_us_per_step": {k: round(v, 1) for k, v in groups.items()},
           "back_share_of_step": round(groups["back"] / (1e3 * step_ms), 4),
           "back_share_of_kernel_time_outside_select": round(groups["back"] / (total_us - groups["select"]), 4),
           "kernels": rows}

    print("%s, power limit / max SM clock: %s" % (name, limit))
    print("workload %s %dx%d K=%d batch %d: %.3f ms per sequential step, %.1f us of kernel time per step"
          % (args.workload, W, H, K, B, step_ms, total_us))
    print("%-18s %-7s %10s %9s %11s %8s" % ("kernel", "group", "us/step", "launches", "of kernels", "of step"))
    for r in rows:
        print("%-18s %-7s %10.1f %9.1f %10.1f%% %7.1f%%" % (r["kernel"], r["group"], r["us_per_step"],
                                                          r["launches_per_step"], 100 * r["share_of_kernel_time"],
                                                          100 * r["share_of_step"]))
    for g, us in groups.items():
        print("%-18s %-7s %10.1f %9s %10.1f%% %7.1f%%" % ("(sum)", g, us, "", 100 * us / total_us,
                                                         100 * us / (1e3 * step_ms)))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
