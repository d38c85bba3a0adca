#!/usr/bin/env python
"""tools/sweep_bench.py — multi-sweep CenterPoint input on an H100: host merge vs device merge vs the streaming ring.

  python tools/sweep_bench.py [--frames N] [--lanes L] [--sweeps K]

A synthetic 20 Hz stream (synth.sweep_sequence: ~29.5k raw points per sweep, the ego driving and turning) feeds the bench
frame (C3 geometry, fp16-pair sparse + dense layers, dense head; bench.py's model) with K = 10 sweeps per frame, ~295k
merged points.  One JSON line per measurement, each with the card name and power limit read in the same run:
  host_merge     (a) io.merge_sweeps per frame on this machine's CPU
  e2e            (b) frames/s of (i) host merge + CenterPointSweep.infer_many, (ii) device merge with every sweep of a
                     frame uploaded, (iii) the streaming ring (one sweep uploaded per frame), each with L lanes;
                 (d) H2D bytes per frame of each mode
  merge_kernel   (c) the merge alone in a CUDA graph: us, algorithmic GB/s, fraction of 3.35 TB/s (H100 SXM data sheet)
  modes_agree    (e) the first frames of the three modes: equal boxes, scores and labels
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bench import BN_GAIN  # noqa: E402
from pointpillars_bench import gpu_identity  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def frame_inputs(seq, j, K):
    from paddle3d_b200 import sweep_ring
    ids = sweep_ring.frame_sweeps(j, K)
    key, pk, tk = seq[ids[0]]
    return key, [(seq[s][0], sweep_ring.ref_from_curr(pk, seq[s][1]), tk - seq[s][2]) for s in ids[1:]]


def host_merge_frames(seq, K, si, cap, pool):
    """Mode (i) input: each frame merged on the host into one of `pool` pinned [cap, F] buffers (reused after the frame's
    result has been read: pool > 2 * lanes)."""
    from paddle3d_b200 import io as p3d_io
    for j in range(len(seq)):
        merged = p3d_io.merge_sweeps(*frame_inputs(seq, j, K), use_dim=si["use_dim"], use_time_lag=si["use_time_lag"],
                                     sweep_remove_radius=si["remove_radius"])
        if len(merged) > cap:
            raise RuntimeError("frame %d: %d merged points exceed the capacity %d" % (j, len(merged), cap))
        h = pool[j % len(pool)].numpy()
        h[:len(merged)] = merged
        h[len(merged):] = np.nan
        yield pool[j % len(pool)]


def reupload_stream(sweep, ring, seq, K):
    """Mode (ii): every frame uploads all of its sweeps again (K pushes), then merges them on the device."""
    from paddle3d_b200.frame import run_in_flight
    for p in sweep.lanes:
        p.prepare_sweep()
    ring.reset()

    def submit(lane, j, _, k):
        ids = list(range(max(0, j - K + 1), j + 1))  # oldest first: the key is the last push
        for s in ids:
            last = ring.push(*seq[s])
        ring.first = last - len(ids) + 1  # the frame reads exactly this frame's uploads
        lane._submit_sweep(last, k)
    yield from run_in_flight(sweep.lanes, range(len(seq)), submit)


def timed(results):
    t0 = time.perf_counter()
    out = [tuple(x.clone() for x in r) for r in results]
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60, help="timed frames per mode (one per sweep of the stream)")
    ap.add_argument("--lanes", type=int, default=4)
    ap.add_argument("--sweeps", type=int, default=10, help="sweeps per frame (K)")
    ap.add_argument("--check", type=int, default=12, help="first frames compared across the three modes")
    args = ap.parse_args()
    import torch

    from paddle3d_b200 import io as p3d_io
    from paddle3d_b200 import synth
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.ops import sweep_merge as sm
    from paddle3d_b200.pipeline import SWEEP_INPUT, CenterPointSweep
    from paddle3d_b200.sweep_ring import SweepRing

    if not torch.cuda.is_available():
        raise SystemExit("sweep_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = gpu_identity(0)
    K, L = args.sweeps, args.lanes
    cfg = synth.C3
    cap = cfg["num_points"]
    seq = synth.sweep_sequence(args.frames + K, 7)
    si = dict(SWEEP_INPUT, max_sweeps=K, slot_cap=-(-max(len(c) for c, _, _ in seq) // 4) * 4)
    cols = sm.columns(si["use_dim"], si["raw_dim"])
    si_cols = dict(si, use_dim=cols)

    def emit(d):
        print(json.dumps(dict(d, gpu=gpu)), flush=True)

    # (a) host merge alone
    t = []
    for j in range(K - 1, len(seq)):
        t0 = time.perf_counter()
        merged = p3d_io.merge_sweeps(*frame_inputs(seq, j, K), use_dim=cols, use_time_lag=True,
                                     sweep_remove_radius=si["remove_radius"])
        t.append(time.perf_counter() - t0)
    emit({"measure": "host_merge", "what": "io.merge_sweeps per %d-sweep frame on the host CPU (numpy)" % K,
          "ms_mean": 1e3 * float(np.mean(t)), "ms_median": 1e3 * float(np.median(t)), "frames": len(t),
          "merged_points": int(len(merged)), "cpu_count": os.cpu_count()})

    # the bench frame, twice: L lanes fed merged clouds, L lanes with the device merge (one model shared by all)
    kw = dict(cfg=cfg, device=dev, precision=sp.F16X3, seed=0, with_head=True, keep_bev=False, bn_gain=BN_GAIN)
    plain = CenterPointSweep(L, **kw)
    ring = SweepRing(K, si["raw_dim"], si["slot_cap"], K * (L + 1), dev)  # room for mode (ii)'s K uploads per frame
    merge = CenterPointSweep(L, sweep_input=si, sweep_ring=ring, **kw)
    for p in merge.lanes:
        p.share_model(plain.lanes[0])
    pool = [torch.empty((cap, 5), dtype=torch.float32).pin_memory() for _ in range(2 * L + 2)]
    dev_first = list(host_merge_frames(seq[:K], K, si_cols, cap, pool[:1]))[-1].to(dev)  # the first full K-sweep frame
    plain.calibrate_head(dev_first)
    plain.capture(dev_first)
    for p in merge.lanes:
        p.infer_sweeps(*frame_inputs(seq, K - 1, K))
        p.capture()

    modes = {
        "host_merge+infer_many": lambda s: plain.infer_many(host_merge_frames(s, K, si_cols, cap, pool)),
        "device_merge_all_sweeps_uploaded": lambda s: reupload_stream(merge, ring, s, K),
        "device_merge_stream_ring": lambda s: merge.infer_stream(iter(s)),
    }
    raw_rows = [len(c) for c, _, _ in seq]
    full = [sum(raw_rows[max(0, j - K + 1):j + 1]) for j in range(len(seq))]
    desc = K * sm.DESC_DTYPE.itemsize
    h2d = {"host_merge+infer_many": cap * 5 * 4,
           "device_merge_all_sweeps_uploaded": float(np.mean(full[K - 1:])) * si["raw_dim"] * 4 + desc,
           "device_merge_stream_ring": float(np.mean(raw_rows)) * si["raw_dim"] * 4 + desc}
    results = {}
    for name, run in modes.items():
        timed(run(seq[:K + 2 * L]))  # warm-up
        out, secs = timed(run(seq))
        results[name] = out
        # (b) + (d)
        emit({"measure": "e2e", "mode": name, "lanes": L, "frames": len(seq), "frames_per_s": len(seq) / secs,
              "h2d_bytes_per_frame": int(h2d[name]),
              "note": "one frame per sweep of the stream; the first K - 1 frames merge fewer sweeps"})

    # (e) the three modes agree.  Bit equality is reported as measured; the fp16-pair frame's last bits follow the
    # (atomics-numbered) row order of the strided sparse levels, so two runs of one cloud may differ there: the labels
    # and the largest box difference over rows with equal labels are reported beside it.
    names = list(results)
    for n in names[1:]:
        eq, same_count, label_match, box_diff = [], [], [], 0.0
        for j in range(min(args.check, len(seq))):
            a, b = results[names[0]][j], results[n][j]
            eq.append(all(torch.equal(x, y) for x, y in zip(a, b)))
            same_count.append(len(a[2]) == len(b[2]))
            if same_count[-1] and len(a[2]):
                keep = (a[2] == b[2]).numpy()
                label_match.append(float(keep.mean()))
                box_diff = max(box_diff, float((a[0].numpy()[keep] - b[0].numpy()[keep]).__abs__().max(initial=0.0)))
        emit({"measure": "modes_agree", "modes": [names[0], n], "frames": len(eq), "bit_equal": eq,
              "same_box_count": all(same_count), "min_label_agreement": min(label_match) if label_match else None,
              "max_abs_box_diff_equal_labels": box_diff})

    # (c) the merge alone, graph-timed on lane 0's buffers (a full K-sweep frame of the stream)
    p = merge.lanes[0]
    p.infer_sweeps(*frame_inputs(seq, len(seq) - 1, K))
    n_raw = sum(len(c) for c in [frame_inputs(seq, len(seq) - 1, K)[0]] +
                [s[0] for s in frame_inputs(seq, len(seq) - 1, K)[1]])
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        run = lambda: sm.merge_into(ring.buf, p._sweep_desc, K, cols, True, si["remove_radius"], p.points,  # noqa: E731
                                    p._n_merged, p._merge_status)
        run()
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        reps = 50
        with torch.cuda.graph(g, stream=st):
            for _ in range(reps):
                run()
        for _ in range(3):
            g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 20
        e0.record(st)
        for _ in range(iters):
            g.replay()
        e1.record(st)
    st.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (iters * reps)
    nbytes = 4 * si["raw_dim"] * n_raw + 4 * 5 * cap
    emit({"measure": "merge_kernel", "what": "merge_sweeps (memset + merge + NaN tail), %d sweeps, %d raw points -> "
          "[%d, 5]" % (K, n_raw, cap), "merged_points": p.merged_rows(), "us": us, "algorithmic_bytes": nbytes,
          "GB_per_s": nbytes / us * 1e-3, "fraction_of_3.35TBps": nbytes / (us * 1e-6) / HBM_BYTES_PER_S})


if __name__ == "__main__":
    main()
