"""soft_slic at the 720p workload: 32 images of 1280x720, K = 1600 (a 30 x 53 grid), C in {20, 64}, n_iter in {5, 10},
features resident in HBM.

Prints, as JSON lines (and, with --out FILE, writes the whole report there as JSON):
  * the card's name, power limit and max SM clock, read in the same run;
  * per (C, n_iter): the forward call's time and the forward + backward time (CUDA events, after warm-up, median of
    --reps), and the peak memory of forward + backward above the inputs;
  * the same for a float32 pure-torch SSN (unfold + softmax + autograd) on --torch-batch images, or "out of memory";
  * image 0 of (C = 20, n_iter = 5) checked bit for bit against the numpy restatement (tests/soft_slic_cases.py);
  * with --profile: the per-kernel times of one forward + backward from torch.profiler (a separate run).
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

B, H, W, K = 32, 720, 1280, 1600


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def features(B, C, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.arange(H, device="cuda", dtype=torch.float32)[:, None]
    x = torch.arange(W, device="cuda", dtype=torch.float32)[None, :]
    a = torch.rand((B, C, 3), generator=g, device="cuda") * 0.05 + 0.005
    f = torch.sin(x * a[..., 0, None, None] + y * a[..., 1, None, None] + a[..., 2, None, None] * 100)
    return (f + torch.randn((B, C, H, W), generator=g, device="cuda") * 0.1).contiguous()


def timed(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def ours(x, n_iter, grads=None):
    from fast_slic_b200.soft_slic import soft_slic
    r = soft_slic(x, K, n_iter)
    if grads is not None:
        torch.autograd.backward([r.assoc, r.centroids], list(grads))
    return r


class TorchSSN:
    """SSN in float32 torch: every iteration unfolds the 3x3 cell neighbourhood of the centroids to every pixel (9*C
    floats per pixel), a dense softmax over the 9 slots, scatter-adds for the weighted means; autograd through all."""

    def __init__(self, grid, dev):
        nh, nw = grid
        self.nh, self.nw = nh, nw
        a = torch.arange(H, device=dev)[:, None] * nh // H
        b = torch.arange(W, device=dev)[None, :] * nw // W
        self.own = (a * nw + b).reshape(-1)
        ks, oks = [], []
        for da in (-1, 0, 1):
            for db in (-1, 0, 1):
                aa, bb = a + da, b + db
                ok = (aa >= 0) & (aa < nh) & (bb >= 0) & (bb < nw)
                ks.append(torch.where(ok, aa * nw + bb, 0).expand(H, W).reshape(-1))
                oks.append(ok.expand(H, W).reshape(-1))
        self.k, self.ok = torch.stack(ks), torch.stack(oks)

    def __call__(self, f, n_iter):
        Bt, C = f.shape[:2]
        nh, nw, Kt = self.nh, self.nw, self.nh * self.nw
        ff = f.reshape(Bt, C, -1)
        cnt = torch.bincount(self.own, minlength=Kt).float()
        mu = torch.zeros(Bt, C, Kt, device=f.device).index_add(2, self.own, ff) / cnt
        for _ in range(n_iter):
            nb = torch.nn.functional.unfold(mu.reshape(Bt, C, nh, nw), 3, padding=1).reshape(Bt, C, 9, Kt)
            mu9 = nb[:, :, :, self.own]                                     # [B,C,9,HW]
            d = (ff[:, :, None] - mu9).square().sum(1)                      # [B,9,HW]
            q = torch.softmax(d.neg().masked_fill(~self.ok, float("-inf")), 1)
            A = torch.zeros(Bt, C, Kt, device=f.device)
            Z = torch.zeros(Bt, Kt, device=f.device)
            for n in range(9):
                A = A.index_add(2, self.k[n], q[:, None, n] * ff)
                Z = Z.index_add(1, self.k[n], q[:, n])
            mu = A / Z[:, None]
        return q, mu


def measure(fn, reps):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    return timed(fn, reps), peak / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--torch-batch", type=int, default=4)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    from fast_slic_b200.soft_slic import cell_grid
    grid = cell_grid(H, W, K)
    report = {"card": card(), "workload": {"B": B, "H": H, "W": W, "K": K, "grid": grid}, "rows": []}
    print(json.dumps(report["card"]), flush=True)

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        x = features(B, 20).requires_grad_(True)
        ga, gc = torch.randn(B, 9, H, W, device="cuda"), torch.randn(B, 20, grid[0] * grid[1], device="cuda")
        ours(x, 5, (ga, gc))
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ours(x, 5, (ga, gc))
            torch.cuda.synchronize()
        rows = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
                t = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
                rows[e.key] = {"ms": t / 1e3, "count": e.count}
        report["profile_c20_iter5"] = dict(sorted(rows.items(), key=lambda kv: -kv[1]["ms"]))
        for k, v in list(report["profile_c20_iter5"].items())[:25]:
            print(json.dumps({"kernel": k[:90], **v}), flush=True)
    else:
        for C in (20, 64):
            x = features(B, C).requires_grad_(True)
            ga = torch.randn(B, 9, H, W, device="cuda")
            gc = torch.randn(B, C, grid[0] * grid[1], device="cuda")
            for n_iter in (5, 10):
                row = {"C": C, "n_iter": n_iter}
                with torch.no_grad():
                    row["forward_ms"] = timed(lambda: ours(x.detach(), n_iter), args.reps)
                row["fwd_bwd_ms"], row["fwd_bwd_peak_gib"] = measure(lambda: ours(x, n_iter, (ga, gc)), args.reps)
                x.grad = None
                tb = args.torch_batch
                ssn = TorchSSN(grid, x.device)
                xt = x[:tb].detach().clone().requires_grad_(True)
                try:
                    with torch.no_grad():
                        row["torch_forward_ms"] = timed(lambda: ssn(xt.detach(), n_iter), args.reps, 1)
                    row["torch_fwd_bwd_ms"], row["torch_fwd_bwd_peak_gib"] = measure(
                        lambda: torch.autograd.backward(list(ssn(xt, n_iter)), [ga[:tb].reshape(tb, 9, -1), gc[:tb]]), args.reps)
                    row["torch_batch"] = tb
                except torch.cuda.OutOfMemoryError:
                    row["torch"] = "out of memory at batch %d" % tb
                del xt
                torch.cuda.empty_cache()
                if C == 20 and n_iter == 5:
                    from soft_slic_cases import nan_class_equal, ref_soft_slic_image
                    from fast_slic_b200.soft_slic import soft_slic
                    r = soft_slic(x.detach(), K, n_iter, min_size_factor=None)
                    lab, q, mu = ref_soft_slic_image(x[0].detach().cpu().numpy(), grid, n_iter)
                    row["image0_bit_exact"] = bool(
                        nan_class_equal(r.assoc[0].cpu().numpy(), q) and nan_class_equal(r.centroids[0].cpu().numpy(), mu)
                        and np.array_equal(r.labels[0].cpu().numpy().astype(np.int64), lab))
                    del r
                report["rows"].append(row)
                print(json.dumps(row), flush=True)
            del x, ga, gc
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
