"""boundary_stats_3d, segmentation_scores_3d and boundaries_3d on supervoxel label volumes, resident in HBM:
  ct     4 volumes of 256 x 512 x 512 (D x H x W), C = 1, K = 16384 (CT-like)
  mri    8 volumes of 155 x 240 x 240, C = 4, K = 4000 (multi-modal MRI-like)
Labels come from supervoxel_slic on the volumes of tools/supervoxel_probe.py; the values of boundary_stats_3d are the
volumes themselves (C channels), the ground truth of the scores is a second supervoxel_slic of the same volumes at
K / 8 (a coarser segmentation), with the tolerance (1, 2, 2).

Prints, as JSON lines (and, with --out FILE, writes the whole report there as JSON):
  * the card's name and power limit, read in the same run;
  * per workload and call: the call time (CUDA events, median of --reps after warm-up), the kernel split of one call
    from torch.profiler (a separate run), and for boundary_stats_3d at 6, 18 and 26 the boundary voxel and pair counts
    and the select and stats scratch bytes;
  * on the workloads named by --torch, the torch route a user writes today, timed the same way: for the statistics
    the boundary pairs per direction, a stable sort of their keys, segment sums / amin / amax with scatter_reduce;
    for the scores shifted compares, max_pool3d for the window and torch.unique for the overlap table.
Every output is checked before anything is printed: count, min and max equal to the torch route and mean within
1e-4 (relative above 1; the values are of order 1 and the torch route sums in float64); the scores and the outline
equal.  Where the torch route does not run, count is checked against region_adjacency_3d's boundary.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from supervoxel_probe import card, kernel_times, timed, volumes  # noqa: E402
from volume_graph_probe import _pairs  # noqa: E402

WORKLOADS = {
    "ct": dict(B=4, C=1, D=256, H=512, W=512, K=16384),
    "mri": dict(B=8, C=4, D=155, H=240, W=240, K=4000),
}
TOLERANCE = (1, 2, 2)


def torch_stats(labels, K, edge_index, values, connectivity):
    """mean, min, max [E,C] and count [E] the torch way (mean in float64, rounded to float32)."""
    from fast_slic_b200.region_graph import RAG3D_OFFSETS
    n = {6: 3, 18: 9, 26: 13}[connectivity]
    lab = labels.long() & 0xFFFF
    B, C = values.shape[:2]
    dev = lab.device
    idx = torch.arange(lab[0].numel(), device=dev).view(lab.shape[1:])
    keys, va, vo = [], [], []
    for (a, c), (ia, io) in zip(_pairs(lab, RAG3D_OFFSETS[:n]), _pairs(idx[None], RAG3D_OFFSETS[:n])):
        ok = (a < K) & (c < K) & (a != c)
        b = torch.arange(B, device=dev).view(B, 1, 1, 1).expand_as(a)[ok]
        keys.append((b * K + torch.minimum(a, c)[ok]) * K + torch.maximum(a, c)[ok])
        flat = values.view(B, C, -1)
        va.append(flat[b, :, ia.expand_as(a)[ok]])
        vo.append(flat[b, :, io.expand_as(a)[ok]])
    key = torch.cat(keys)
    v = torch.cat([torch.cat(va), torch.cat(vo)])  # [2P, C]
    u, inv, cnt = torch.unique(key, return_inverse=True, return_counts=True)
    inv2 = torch.cat([inv, inv])
    R = u.numel()
    s = torch.zeros((R, C), dtype=torch.float64, device=dev).index_add_(0, inv2, v.double())
    mn = torch.full((R, C), float("inf"), device=dev).scatter_reduce_(0, inv2[:, None].expand_as(v), v, "amin")
    mx = torch.full((R, C), -float("inf"), device=dev).scatter_reduce_(0, inv2[:, None].expand_as(v), v, "amax")
    u_src, u_dst = edge_index
    bsrc = u_src // K
    ekey = (bsrc * K + torch.minimum(u_src % K, u_dst % K)) * K + torch.maximum(u_src % K, u_dst % K)
    at = torch.searchsorted(u, ekey).clamp_max(R - 1)
    hit = u[at] == ekey
    E = edge_index.shape[1]
    nan = torch.full((E, C), float("nan"), device=dev)
    mean = torch.where(hit[:, None], (s[at] / (2 * cnt[at, None]).double()).float(), nan)
    return mean, torch.where(hit[:, None], mn[at], nan), torch.where(hit[:, None], mx[at], nan), \
        torch.where(hit, cnt[at], 0).int()


def _outline(lab):
    out = torch.zeros_like(lab, dtype=torch.bool)
    out[..., :-1] |= lab[..., :-1] != lab[..., 1:]
    out[..., :-1, :] |= lab[..., :-1, :] != lab[..., 1:, :]
    out[..., :-1, :, :] |= lab[..., :-1, :, :] != lab[..., 1:, :, :]
    return out


def torch_scores(labels, gt, K, tol):
    """The seven integer fields [B,7] the torch way."""
    B = labels.shape[0]
    lab = labels.long() & 0xFFFF
    g = gt.long()
    ok = g >= 0
    sp = _outline(lab)
    e = torch.zeros_like(sp)
    for axis in (3, 2, 1):
        a = [slice(None)] * 4
        c = list(a)
        a[axis], c[axis] = slice(None, -1), slice(1, None)
        a, c = tuple(a), tuple(c)
        e[a] |= ok[a] & ok[c] & (g[a] != g[c])
    rz, ry, rx = tol
    size = (2 * rz + 1, 2 * ry + 1, 2 * rx + 1)
    ds, de = (F.max_pool3d(m[:, None].half(), size, 1, (rz, ry, rx))[:, 0] > 0 for m in (sp, e))
    counted = ok & (lab < K)
    out = torch.zeros((B, 7), dtype=torch.int64, device=lab.device)
    for b in range(B):
        key = lab[b][counted[b]] * 2 ** 31 + g[b][counted[b]]
        u, n_kg = torch.unique(key, return_counts=True)
        k_of = u // 2 ** 31
        n_k = torch.zeros(K, dtype=torch.int64, device=lab.device).index_add_(0, k_of, n_kg)
        mx = torch.zeros(K, dtype=torch.int64, device=lab.device).scatter_reduce_(0, k_of, n_kg, "amax")
        out[b, 0], out[b, 1] = counted[b].sum(), mx.sum()
        out[b, 2] = torch.minimum(n_kg, n_k[k_of] - n_kg).sum()
    out[:, 3] = e.flatten(1).sum(1)
    out[:, 4] = (e & ds).flatten(1).sum(1)
    out[:, 5] = (sp & ok).flatten(1).sum(1)
    out[:, 6] = (sp & ok & de).flatten(1).sum(1)
    return out


def select_counts(labels, K, connectivity):
    """(boundary voxels, boundary pairs) of int16 [B,D,H,W] labels: the select step of boundary_stats_3d alone."""
    from fast_slic_b200 import _lib
    L = _lib.lib()
    B, D, H, W = labels.shape
    nbytes = int(L.fslic_b200_boundary3d_select_scratch_bytes(B, D, H, W, K, connectivity))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=labels.device)
    counts = torch.empty(2, dtype=torch.int64, device=labels.device)
    _lib.check(L.fslic_b200_boundary3d_select_batch(labels.device.index, B, D, H, W, K, connectivity,
                                                    labels.contiguous().data_ptr(), counts.data_ptr(),
                                                    scratch.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream))
    return tuple(counts.tolist())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="mri,ct")
    ap.add_argument("--torch", default="mri", help="workloads on which the torch routes run and are timed")
    ap.add_argument("--compactness", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the whole report to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("volume_boundary_probe needs a CUDA device")
    from fast_slic_b200 import _lib
    from fast_slic_b200.groundtruth import boundaries_3d, segmentation_scores_3d
    from fast_slic_b200.region_graph import boundary_stats_3d, region_adjacency_3d
    from fast_slic_b200.supervoxels import supervoxel_slic
    L = _lib.lib()
    report = {"card": card()}
    print(json.dumps(report["card"]), flush=True)
    rows = []
    for name in a.workloads.split(","):
        w = WORKLOADS[name]
        B, C, D, H, W, K = w["B"], w["C"], w["D"], w["H"], w["W"], w["K"]
        x = volumes(B, C, D, H, W, seed=len(rows))
        r = supervoxel_slic(x, K, a.compactness)
        labels, K2 = r.labels, int(r.position.shape[1])
        gt = supervoxel_slic(x, K // 8, a.compactness).labels.int()
        del r
        torch.cuda.empty_cache()
        use_torch = name in a.torch.split(",")
        row = {"workload": name, **w, "K_prime": K2, "calls": []}
        for conn in (6, 18, 26):
            g = region_adjacency_3d(labels, K2, conn)
            run = lambda: boundary_stats_3d(labels, K2, g, x, conn)  # noqa: E731
            out = run()
            if not torch.equal(out.count, g.boundary):
                sys.exit("boundary_stats_3d %d on %s: count differs from the graph's boundary" % (conn, name))
            entry = {"call": "boundary_stats_3d", "connectivity": conn, "edges": int(g.edge_index.shape[1])}
            if use_torch:
                ref = torch_stats(labels, K2, g.edge_index, x, conn)
                same = (torch.equal(out.count, ref[3]) and torch.equal(out.min, ref[1]) and torch.equal(out.max, ref[2])
                        and bool(((out.mean - ref[0]).abs() <= 1e-4 * ref[0].abs().clamp_min(1)).all()))
                if not same:
                    sys.exit("boundary_stats_3d %d on %s: outputs differ from the torch route" % (conn, name))
                del ref
                entry["checked"] = "count, min, max equal to the torch route, mean within 1e-4"
            else:
                entry["checked"] = "count equal to region_adjacency_3d's boundary"
            # the boundary voxel and pair counts of the batch and of each volume, and the scratch they need
            voxels, pairs = select_counts(labels, K2, conn)
            per = [select_counts(labels[b:b + 1], K2, conn) for b in range(B)]
            E = int(g.edge_index.shape[1])
            entry.update(voxels=B * D * H * W, boundary_voxels=voxels, boundary_pairs=pairs,
                         pairs_per_voxel=pairs / (B * D * H * W), per_volume_pairs_max=max(p for _, p in per),
                         select_scratch_bytes=int(L.fslic_b200_boundary3d_select_scratch_bytes(B, D, H, W, K2, conn)),
                         stats_scratch_bytes=int(L.fslic_b200_boundary3d_stats_scratch_bytes(voxels, pairs, E)),
                         single_volume_stats_scratch_bytes=max(
                             int(L.fslic_b200_boundary3d_stats_scratch_bytes(v, p, E)) for v, p in per))
            del out
            torch.cuda.empty_cache()
            med, lo, hi = timed(run, a.reps, a.warmup)
            entry["call_ms"], entry["call_ms_min_max"] = med, [lo, hi]
            kt = kernel_times(run)
            entry["kernels_ms"] = {k: round(sum(v), 4) for k, v in sorted(kt.items(), key=lambda kv: -sum(kv[1]))}
            if use_torch:
                entry["torch_route_ms"] = timed(lambda: torch_stats(labels, K2, g.edge_index, x, conn), 3, 1)[0]
                entry["speedup_vs_torch"] = entry["torch_route_ms"] / entry["call_ms"]
                torch.cuda.empty_cache()
            print(json.dumps({"workload": name, **entry}), flush=True)
            row["calls"].append(entry)
            del g
            torch.cuda.empty_cache()
        for call in ("segmentation_scores_3d", "boundaries_3d"):
            if call == "segmentation_scores_3d":
                run = lambda: segmentation_scores_3d(labels, gt, K2, TOLERANCE)  # noqa: E731
                got = torch.stack(run()[:7], 1)
                want = torch_scores(labels, gt, K2, TOLERANCE)
            else:
                run = lambda: boundaries_3d(labels)  # noqa: E731
                got, want = run(), _outline(labels.long() & 0xFFFF)
            if not torch.equal(got, want):
                sys.exit("%s on %s: outputs differ from the torch route" % (call, name))
            entry = {"call": call, "checked": "equal to the torch route"}
            if call == "segmentation_scores_3d":
                entry["tolerance"] = TOLERANCE
                entry["scratch_bytes"] = int(L.fslic_b200_gt_scores3d_scratch_bytes(B, D, H, W, K2))
                entry["boundary_recall"] = (got[:, 4].sum() / got[:, 3].sum()).item()
            del got, want
            torch.cuda.empty_cache()
            med, lo, hi = timed(run, a.reps, a.warmup)
            entry["call_ms"], entry["call_ms_min_max"] = med, [lo, hi]
            kt = kernel_times(run)
            entry["kernels_ms"] = {k: round(sum(v), 4) for k, v in sorted(kt.items(), key=lambda kv: -sum(kv[1]))}
            if use_torch:
                tr = (lambda: torch_scores(labels, gt, K2, TOLERANCE)) if call == "segmentation_scores_3d" else \
                    (lambda: _outline(labels.long() & 0xFFFF))
                entry["torch_route_ms"] = timed(tr, 3, 1)[0]
                entry["speedup_vs_torch"] = entry["torch_route_ms"] / entry["call_ms"]
            torch.cuda.empty_cache()
            print(json.dumps({"workload": name, **entry}), flush=True)
            row["calls"].append(entry)
        rows.append(row)
        del x, labels, gt
        torch.cuda.empty_cache()
    report["workloads"] = rows
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
