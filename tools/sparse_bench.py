#!/usr/bin/env python
"""Per-layer timing of the 20 tensor-core sparse convs of SparseResNet3D on frame 0 of the bench (synth.lidar_cloud(C3, 0),
seeded weights, BN gain as in bench.py).

The rulebooks are built once (voxelize + SparseResNet3D.forward_sparse); then every fp16-pair conv launch is graph-timed
alone on its real neighbour map and device row count.  One JSON line per layer: channels, K, rows, 128-row tiles, pairs
(valid neighbour entries), the work decomposition the wgmma kernel chooses on the device (recomputed here from the row
count), microseconds, algorithmic GFLOP (2 * pairs * Cin * Cout) and TFLOP/s, the bytes gathered (pairs * 4 * Cin), the
weight bytes streamed into shared memory (sum over the CTAs' items of taps * 4 * Cin * Cout) and the least time either
bound allows: flops at a third of the data sheet's 989 TFLOP/s (three fp16 MMAs per product), bytes at L2_BYTES_PER_S.
Then the sums over the wgmma layers (csrc/sparse_conv_f16.cu) and the warp-MMA layers (csrc/sparse_conv_wm.cu), and the
whole forward_sparse graph-timed.  Needs a GPU:
    python tools/sparse_bench.py [> sparse_layers.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KM = 128                    # rows of a tile (tc::kM)
MAX_SPLITS = 4              # f16::kMaxSplits
SK_FIX = 6                  # f16::kSkFix
PEAK_FP16_FLOPS = 989e12    # H100 SXM data sheet, dense fp16
L2_BYTES_PER_S = 5.5e12     # assumed L2 -> SM rate of the whole card; stated, not measured here


def choose_splits(n_tiles, grid, K, smax):
    smax = max(1, min(smax, K))
    best, best_cost = 1, None
    for s in range(1, smax + 1):
        waves = (n_tiles * s + grid - 1) // grid
        cost = waves * ((K + s - 1) // s + 4 + (1 if s > 1 else 0))
        if best_cost is None or cost < best_cost:
            best, best_cost = s, cost
    return best


def decomposition(rows, K, grid, smax=MAX_SPLITS):
    """What f16::make_sched chooses for `rows` output rows on `grid` CTAs: kind, pieces per tile, items and taps of the
    busiest CTA."""
    n_tiles = (rows + KM - 1) // KM
    if n_tiles == 0:
        return dict(kind="empty", splits=1, items_per_cta=0, taps_per_cta=0)
    splits = choose_splits(n_tiles, grid, K, smax)
    n_work = n_tiles * splits
    waves = (n_work + grid - 1) // grid
    cost_old = waves * ((K + splits - 1) // splits + 4 + (1 if splits > 1 else 0))
    total = n_tiles * K
    if smax >= 4:
        u_min = max(1, (K - 1 + 2) // 3)
        g = max(1, min(grid, total // u_min))
        per = (total + g - 1) // g
        if per + 4 + SK_FIX < cost_old:
            items = max(((c + 1) * total // g - 1) // K - (c * total // g) // K + 1 for c in range(g))
            return dict(kind="stream-K", splits=0, ctas=g, items_per_cta=items, taps_per_cta=per)
    return dict(kind="split" if splits > 1 else "no split", splits=splits, ctas=min(grid, n_work), items_per_cta=waves,
                taps_per_cta=waves * ((K + splits - 1) // splits))


def counts(cin, cout, K, rows, pairs, grid):
    """Algorithmic work of one layer and the time its two bounds allow."""
    n_tiles = (rows + KM - 1) // KM
    flops = 2.0 * pairs * cin * cout
    gathered = pairs * 4 * cin
    weights = n_tiles * K * 4 * cin * cout  # every (tile, tap) unit streams its Cin x Cout fp16-pair block once
    t_flops = flops / (PEAK_FP16_FLOPS / 3) * 1e6
    t_bytes = (gathered + weights) / L2_BYTES_PER_S * 1e6
    d = decomposition(rows, K, grid)
    return dict(tiles=n_tiles, pairs=int(pairs), decomposition=d, gflop=round(flops / 1e9, 3),
                gathered_mb=round(gathered / 1e6, 2), weight_mb=round(weights / 1e6, 2),
                bound_us=round(max(t_flops, t_bytes), 1), bound="flops" if t_flops > t_bytes else "bytes")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def graph_time(fn, iters=20):
    import torch
    st = torch.cuda.current_stream()
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    best = None
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        g.replay()
        b.record(st)
        b.synchronize()
        us = a.elapsed_time(b) / iters * 1e3
        best = us if best is None or us < best else best
    return best


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--counts", metavar="CIN,COUT,K,ROWS,PAIRS", help="print the host-side counts of one layer and exit "
                    "(no GPU needed)")
    args = ap.parse_args()
    if args.counts:
        cin, cout, K, rows, pairs = [int(v) for v in args.counts.split(",")]
        print(json.dumps(counts(cin, cout, K, rows, pairs, 132)))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("sparse_bench.py needs a CUDA device: it times kernels and has no CPU path")
    from bench import BN_GAIN
    from paddle3d_b200 import synth
    from paddle3d_b200.layers import SparseResNet3D
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.ops import voxelize as vox

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    grid = torch.cuda.get_device_properties(dev).multi_processor_count
    print(json.dumps({"card": card(), "sms": grid, "l2_bytes_per_s_assumed": L2_BYTES_PER_S}), flush=True)

    cfg = synth.C3
    V = cfg["max_voxels"]
    net = SparseResNet3D(cfg["point_dim"], cfg["voxel_size"], cfg["point_cloud_range"])
    net.init_weight(seed=0, device=dev, bn_gain=BN_GAIN).set_precision(sp.F16X3).set_level_caps([3 * V, 3 * V, 2 * V, V])
    pts = torch.from_numpy(synth.lidar_cloud(cfg, 0)).to(dev)

    def forward():
        mean, coors, _, nv = vox.voxelize_mean(pts, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"],
                                               cfg["max_voxels"], 0)
        out, _ = net.forward_sparse(mean, coors, 1, num=nv)
        return out.get(sp.ROWS_H16)

    # record every fused launch of one forward: (pending kernel, layout it was asked for)
    launches = []
    run = sp._run

    def recording_run(p, t, want):
        run(p, t, want)  # its inputs launch first: the list is in execution order
        launches.append((p, want))
    sp._run = recording_run
    forward()
    sp._run = run
    torch.cuda.synchronize()

    sums = {"wgmma": 0.0, "wm": 0.0}
    for i, (p, want) in enumerate(launches):
        if p.precision != sp.F16X3:
            continue
        rows = min(int(p.num[0].item()), p.cap)
        pairs = int((p.nbr[:rows] >= 0).sum().item())
        kern = "wm" if p.wm else "wgmma"
        row = {"layer": i, "kernel": kern, "cin": p.cin, "cout": p.cout, "K": p.K, "rows": rows,
               "residual": p.residual is not None}
        row.update(counts(p.cin, p.cout, p.K, rows, pairs, grid))
        if p.wm:
            del row["decomposition"]  # the warp-MMA kernel has its own stream-K
        sink = sp.SparseCooTensor(p.x.index, channels=p.cout)
        us = graph_time(lambda: run(p, sink, want))
        sums[kern] += us
        row.update(us=round(us, 1), algorithmic_tflops=round(row["gflop"] / us * 1e3, 1),
                   share_of_bound=round(row["bound_us"] / us, 3))
        print(json.dumps(row), flush=True)
    print(json.dumps({"wgmma_layers_us": round(sums["wgmma"], 1), "wm_layers_us": round(sums["wm"], 1),
                      "forward_sparse_us": round(graph_time(forward, 5), 1)}), flush=True)


if __name__ == "__main__":
    main()
