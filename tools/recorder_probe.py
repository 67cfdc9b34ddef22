"""Cost of debug_mode at 1280x720, K=1600, 10 iterations (DESIGN.md section 4.11).

Times on one Engine, device buffers, the context's own stream:
  * iterate with tracing off, and on (both end in a device synchronise): the difference is the GPU capture -- one
    trace kernel per pass, the cluster copies and the unfused prepares;
  * trace_snapshots (device -> host copy of one image's snapshots) and format_recorder_report (host text) separately;
  * the report size, and the compiled reference's time for the same report (oracle/_ref, where built).
Prints one JSON line with the device name and power limit beside the numbers.

    python tools/recorder_probe.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fast_slic_b200 import Engine, _lib  # noqa: E402
from oracle.oracle import Port, synthetic_image  # noqa: E402
from oracle.recorder import RecorderRef  # noqa: E402


def _gpu_line():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    H, W, K, it = 720, 1280, 1600, 10
    img = synthetic_image(H, W, seed=11)
    eng = Engine(H, W, K, max_batch=1)
    st = torch.cuda.Stream()
    d_img = torch.from_numpy(img).cuda()[None]
    params = Engine.params(10.0, 0.25, 3, True, it)
    seeds = eng.initialize_clusters(d_img)
    torch.cuda.synchronize()

    def run(trace):
        cl = seeds.clone()
        torch.cuda.synchronize()
        eng.set_trace(trace)
        t0 = time.perf_counter()
        with torch.cuda.stream(st):
            eng.iterate(d_img, cl, params)
        st.synchronize()
        t1 = time.perf_counter()
        eng.set_trace(False)
        return (t1 - t0) * 1e3

    res = {"off": [], "on": [], "d2h": [], "format": []}
    for trace in (False, True, False, True):  # warm-up of both shapes
        run(trace)
    for _ in range(args.reps):
        res["off"].append(run(False))
        res["on"].append(run(True))
        t0 = time.perf_counter()
        s = eng.trace_snapshots(0)
        t1 = time.perf_counter()
        rep = _lib.format_recorder_report(H, W, s["assignment"], s["min_dists"], s["clusters"])
        t2 = time.perf_counter()
        res["d2h"].append((t1 - t0) * 1e3)
        res["format"].append((t2 - t1) * 1e3)
    out = {k + "_ms_median": float(np.median(v)) for k, v in res.items()}
    out["report_bytes"] = len(rep)
    out["mismatches"] = s["mismatches"]
    if RecorderRef.available():
        ref = RecorderRef()
        times = []
        for _ in range(2):
            cl = Port().initialize(img, K)
            t0 = time.perf_counter()
            ref_rep, _ = ref.iterate("standard", img, cl, max_iter=it, num_threads=-1)
            times.append((time.perf_counter() - t0) * 1e3)
        out["reference_ms_median"] = float(np.median(times))
        out["reference_report_equal"] = ref_rep == rep
        out["host_cpus"] = os.cpu_count()
    else:
        out["reference_ms_median"] = None
    out["gpu"] = _gpu_line()
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
