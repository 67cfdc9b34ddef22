"""region_adjacency_3d and region_properties_3d on supervoxel label volumes, resident in HBM:
  ct     4 volumes of 256 x 512 x 512 (D x H x W), C = 1, K = 16384 (CT-like)
  mri    8 volumes of 155 x 240 x 240, C = 4, K = 4000 (multi-modal MRI-like)
Labels come from supervoxel_slic on the volumes of tools/supervoxel_probe.py.

Prints, as JSON lines (and, with --out FILE, writes the whole report there as JSON):
  * the card's name and power limit, read in the same run;
  * per workload: supervoxel_slic's call time; per call and connectivity the call time (CUDA events, median of --reps
    after warm-up), its share of supervoxel_slic's time in the same process, the kernel split of one call from
    torch.profiler (a separate run), the edge count, the largest pair-table load and the volumes counted again after
    an overflow;
  * on the workloads named by --torch, the torch route a user writes today, timed the same way: for the graph the keys
    of the valid differing voxel pairs, torch.unique(return_counts=True), both directions, argsort, bincount + cumsum;
    for the shapes scatter_add_ / scatter_reduce and shifted compares.
Every output is checked before anything is printed: against the torch route where it runs; elsewhere the graph's
boundary total against torch's count of differing valid voxel pairs and its symmetry, and the shapes' area against
torch.bincount.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from supervoxel_probe import card, kernel_times, volumes  # noqa: E402

WORKLOADS = {
    "ct": dict(B=4, C=1, D=256, H=512, W=512, K=16384),
    "mri": dict(B=8, C=4, D=155, H=240, W=240, K=4000),
}


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
    return statistics.median(ms)


def _pairs(lab, offsets):
    """(anchor, neighbour) label views of [B,D,H,W] for each forward offset."""
    _, D, H, W = lab.shape
    for o in offsets:
        sa = [slice(max(0, -v), L - max(0, v)) for L, v in zip((D, H, W), o)]
        sc = [slice(max(0, v), L + min(0, v)) for L, v in zip((D, H, W), o)]
        yield lab[:, sa[0], sa[1], sa[2]], lab[:, sc[0], sc[1], sc[2]]


def torch_rag3d(labels, K, connectivity):
    from fast_slic_b200.region_graph import RAG3D_OFFSETS
    n = {6: 3, 18: 9, 26: 13}[connectivity]
    lab = labels.long() & 0xFFFF
    B = lab.shape[0]
    keys = []
    for a, c in _pairs(lab, RAG3D_OFFSETS[:n]):
        ok = (a < K) & (c < K) & (a != c)
        b = torch.arange(B, device=lab.device).view(B, 1, 1, 1).expand_as(a)[ok]
        keys.append((b * K + torch.minimum(a, c)[ok]) * K + torch.maximum(a, c)[ok])
    u, cnt = torch.unique(torch.cat(keys), return_counts=True)
    b, lo, hi = u // (K * K), u // K % K, u % K
    src = torch.cat([b * K + lo, b * K + hi])
    dst = torch.cat([b * K + hi, b * K + lo])
    order = torch.argsort(src * (B * K) + dst)
    src, dst, w = src[order], dst[order], torch.cat([cnt, cnt])[order].int()
    indptr = torch.zeros(B * K + 1, dtype=torch.int64, device=lab.device)
    indptr[1:] = torch.cumsum(torch.bincount(src, minlength=B * K), 0)
    return indptr, torch.stack([src, dst]), w


def torch_props3d(labels, K):
    lab = labels.long() & 0xFFFF
    B, D, H, W = lab.shape
    dev = lab.device
    ok = lab < K
    node = (torch.arange(B, device=dev).view(B, 1, 1, 1) * K + lab)[ok]
    z = torch.arange(D, device=dev).view(1, D, 1, 1).expand(B, D, H, W)[ok]
    y = torch.arange(H, device=dev).view(1, 1, H, 1).expand(B, D, H, W)[ok]
    x = torch.arange(W, device=dev).view(1, 1, 1, W).expand(B, D, H, W)[ok]
    N = B * K
    add = lambda v: torch.zeros(N, dtype=torch.int64, device=dev).scatter_add_(0, node, v)  # noqa: E731
    area = add(torch.ones_like(node))
    moments = torch.stack([add(v) for v in (z, y, x, z * z, z * y, z * x, y * y, y * x, x * x)], 1)
    big = torch.iinfo(torch.int64).max
    lo = [torch.full((N,), big, device=dev).scatter_reduce_(0, node, v, "amin") for v in (z, y, x)]
    hi = [torch.full((N,), -1, device=dev).scatter_reduce_(0, node, v + 1, "amax") for v in (z, y, x)]
    bbox = torch.stack(lo + hi, 1)
    bbox[area == 0] = 0
    pad = torch.full((B, D + 2, H + 2, W + 2), -1, dtype=torch.int64, device=dev)
    pad[:, 1:-1, 1:-1, 1:-1] = lab
    edge = torch.ones((D + 2, H + 2, W + 2), dtype=torch.int64, device=dev)
    edge[1:-1, 1:-1, 1:-1] = 0
    diff = torch.zeros_like(lab)
    bord = torch.zeros((D, H, W), dtype=torch.int64, device=dev)
    for dz, dy, dx in ((-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)):
        diff += pad[:, 1 + dz:D + 1 + dz, 1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx] != lab
        bord += edge[1 + dz:D + 1 + dz, 1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx]
    surface = add(diff[ok])
    border = add(bord.expand(B, D, H, W)[ok])
    n = area.double().clamp_min(1)[:, None]
    q = moments.double() / n
    c = q[:, :3]
    cov = torch.stack([q[:, f] - c[:, a] * c[:, b] for f, a, b in
                       ((3, 0, 0), (4, 0, 1), (5, 0, 2), (6, 1, 1), (7, 1, 2), (8, 2, 2))], 1)
    c = c.clone()
    c[area == 0] = 0.0
    cov[area == 0] = 0.0
    return (area.int().view(B, K), bbox.int().view(B, K, 6), moments.view(B, K, 9), surface.view(B, K),
            border.int().view(B, K), c.view(B, K, 3), cov.view(B, K, 6))


def _equal(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and torch.equal(x, y) for x, y in zip(a, b))


def graph_checks(g, labels, K, connectivity):
    """The boundary total against torch's count of differing valid voxel pairs, and the graph's symmetry."""
    from fast_slic_b200.region_graph import RAG3D_OFFSETS
    n = {6: 3, 18: 9, 26: 13}[connectivity]
    lab = labels.long() & 0xFFFF
    total = sum(int(((a < K) & (c < K) & (a != c)).sum()) for a, c in _pairs(lab, RAG3D_OFFSETS[:n]))
    N = labels.shape[0] * K
    fwd = g.edge_index[0] * N + g.edge_index[1]
    rev = g.edge_index[1] * N + g.edge_index[0]
    order = torch.argsort(rev)
    return (int(g.boundary.long().sum()) == 2 * total and torch.equal(rev[order], fwd)
            and torch.equal(g.boundary[order], g.boundary))


def props_checks(p, labels, K):
    B = labels.shape[0]
    lab = (labels.long() & 0xFFFF).clamp_max(K) + torch.arange(B, device=labels.device).view(B, 1, 1, 1) * (K + 1)
    cnt = torch.bincount(lab.view(-1), minlength=B * (K + 1)).view(B, K + 1)[:, :K]  # bin K: labels >= K
    return torch.equal(p.area.long(), cnt)


def table_load(g, B, K, D, H, W, connectivity):
    """Largest keys / slots over the volumes of the graph-sized table (what the count uses unless exact is smaller)."""
    from fast_slic_b200.region_graph import voxel_pairs
    t_graph = 4096
    while t_graph < 32 * K:
        t_graph *= 2
    need = 2 * min(K * (K - 1) // 2, voxel_pairs(D, H, W, connectivity))
    t_exact = 1 << max(0, (need - 1).bit_length())
    T = min(t_graph, t_exact)
    per = g.indptr[::K].diff() // 2  # undirected edges of each volume
    return float(per.max()) / T, T


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
        sys.exit("volume_graph_probe needs a CUDA device")
    from fast_slic_b200 import region_graph
    from fast_slic_b200.geometry import region_properties_3d
    from fast_slic_b200.region_graph import region_adjacency_3d
    from fast_slic_b200.supervoxels import supervoxel_slic
    recounts = []
    split = region_graph._split

    def spy(b0, flags):
        recounts.append(sum(flags))
        return split(b0, flags)

    region_graph._split = spy
    report = {"card": card()}
    print(json.dumps(report["card"]), flush=True)
    rows = []
    for name in a.workloads.split(","):
        w = WORKLOADS[name]
        B, C, D, H, W, K = w["B"], w["C"], w["D"], w["H"], w["W"], w["K"]
        x = volumes(B, C, D, H, W, seed=len(rows))
        sv = lambda: supervoxel_slic(x, K, a.compactness)  # noqa: E731
        sv_ms = timed(sv, a.reps, a.warmup)
        r = sv()
        labels, K2 = r.labels, int(r.position.shape[1])
        del r
        torch.cuda.empty_cache()
        row = {"workload": name, **w, "K_prime": K2, "supervoxel_slic_ms": sv_ms, "calls": []}
        use_torch = name in a.torch.split(",")
        calls = [("region_adjacency_3d", c) for c in (6, 18, 26)] + [("region_properties_3d", None)]
        for call, conn in calls:
            if call == "region_adjacency_3d":
                run = lambda: region_adjacency_3d(labels, K2, conn)  # noqa: E731
            else:
                run = lambda: region_properties_3d(labels, K2)  # noqa: E731
            del recounts[:]
            out = run()
            entry = {"call": call, "connectivity": conn, "overflow_recounts": sum(recounts)}
            if use_torch:
                ref = torch_rag3d(labels, K2, conn) if conn else torch_props3d(labels, K2)
                ok = _equal(out, ref)
                del ref
            else:
                ok = graph_checks(out, labels, K2, conn) if conn else props_checks(out, labels, K2)
            if not ok:
                sys.exit("%s %s on %s: outputs differ" % (call, conn, name))
            entry["checked"] = "equal to the torch route" if use_torch else "consistency checks"
            if conn:
                entry["edges"] = int(out.edge_index.shape[1])
                entry["largest_table_load"], entry["table_slots"] = table_load(out, B, K2, D, H, W, conn)
            del out
            torch.cuda.empty_cache()
            entry["call_ms"] = timed(run, a.reps, a.warmup)
            entry["share_of_supervoxel_slic"] = entry["call_ms"] / sv_ms
            kt = kernel_times(run)
            entry["kernels_ms"] = {k: round(sum(v), 4) for k, v in sorted(kt.items(), key=lambda kv: -sum(kv[1]))}
            if use_torch:
                tr = (lambda: torch_rag3d(labels, K2, conn)) if conn else (lambda: torch_props3d(labels, K2))
                entry["torch_route_ms"] = timed(tr, max(5, a.reps // 2), 1)
                entry["speedup_vs_torch"] = entry["torch_route_ms"] / entry["call_ms"]
                torch.cuda.empty_cache()
            print(json.dumps({"workload": name, **entry}), flush=True)
            row["calls"].append(entry)
        rows.append(row)
        del x, labels
        torch.cuda.empty_cache()
    region_graph._split = split
    report["workloads"] = rows
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
