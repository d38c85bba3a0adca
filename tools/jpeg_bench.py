"""Device JPEG decode (ops/jpeg.jpeg_decode_u8) on six nuScenes-sized camera files (synth.camera_jpegs, Pillow q95 4:2:0
unless --quality / --subsampling say otherwise), against Pillow's host decode of the same files in the same run.

Reports, as one JSON line: the captured decode of the six images per frame (whole images and BEVDet's prep band),
timed by CUDA events over graph replays; each kernel's share from torch.profiler; compressed MB/s and output GB/s;
the H2D copy of the compressed bytes from pinned memory next to that of the uint8 band it replaces; the host marker
parse per frame; Pillow's decode of the six files on one thread and on every core; and the card name and power limit
read in the same run."""
import argparse
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quality", type=int, default=95)
    ap.add_argument("--subsampling", type=int, default=2)
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    from PIL import Image

    from paddle3d_b200 import bevdet, synth
    from paddle3d_b200.ops import jpeg
    from paddle3d_b200.ops.image_prep import ImagePrepPlan

    dev = torch.device("cuda:0")
    frames = [synth.camera_jpegs(s, quality=args.quality, subsampling=args.subsampling) for s in range(args.frames)]
    n, H, W = 6, 900, 1600
    cap = max(len(f) for fr in frames for f in fr)
    plan = ImagePrepPlan.from_data_config(bevdet.DATA_CONFIG, device=dev)
    res = dict(card=card(), quality=args.quality, subsampling=args.subsampling,
               compressed_mb_per_frame=float(np.mean([sum(len(f) for f in fr) for fr in frames])) / 1e6)

    # host: marker parse, Pillow decode on one thread and on every core
    t0 = time.perf_counter()
    for fr in frames:
        jpeg.batch(fr)
    res["host_parse_ms_per_frame"] = (time.perf_counter() - t0) * 1e3 / len(frames)

    def pil(f):
        return np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))

    t0 = time.perf_counter()
    for fr in frames:
        for f in fr:
            pil(f)
    res["pillow_one_thread_ms_per_frame"] = (time.perf_counter() - t0) * 1e3 / len(frames)
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        list(ex.map(pil, frames[0]))
        t0 = time.perf_counter()
        for fr in frames:
            list(ex.map(pil, fr))
        res["pillow_all_cores_ms_per_frame"] = (time.perf_counter() - t0) * 1e3 / len(frames)
    res["cpu_count"] = os.cpu_count()

    data_dev = torch.zeros(n * cap, dtype=torch.uint8, device=dev)
    desc_dev = torch.zeros(n * jpeg.DESC_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    status = torch.zeros(n, dtype=torch.int32, device=dev)
    staged = []
    for fr in frames:
        data, desc, _ = jpeg.batch(fr)
        staged.append((torch.from_numpy(data).pin_memory(), torch.from_numpy(desc.view(np.uint8)).pin_memory()))

    def stage(i):
        d, s = staged[i % len(staged)]
        data_dev[:d.numel()].copy_(d, non_blocking=True)
        desc_dev.copy_(s, non_blocking=True)

    for name, rows in (("full", (0, H)), ("band", plan.band)):
        out = torch.empty((n, rows[1] - rows[0], W, 3), dtype=torch.uint8, device=dev)
        stage(0)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            jpeg.jpeg_decode_u8(data_dev, desc_dev, n, (H, W), rows=rows, out=out, status=status, max_bytes=cap)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            jpeg.jpeg_decode_u8(data_dev, desc_dev, n, (H, W), rows=rows, out=out, status=status, max_bytes=cap)
        # correctness of frame 0 against Pillow before timing
        g.replay()
        torch.cuda.synchronize()
        assert not status.any()
        got = out.cpu().numpy()
        for i, f in enumerate(frames[0]):
            assert np.array_equal(got[i], pil(f)[rows[0]:rows[1]]), "frame 0 image %d differs from Pillow" % i
        times = []
        for r in range(args.reps):
            stage(r)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        med = float(np.median(times))
        res["decode_" + name] = dict(rows=list(rows), median_us=med * 1e3, min_us=float(np.min(times)) * 1e3,
                                     compressed_mb_s=res["compressed_mb_per_frame"] / (med * 1e-3),
                                     output_gb_s=out.numel() / (med * 1e-3) / 1e9)
        # per-kernel times of the eager decode
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for r in range(10):
                jpeg.jpeg_decode_u8(data_dev, desc_dev, n, (H, W), rows=rows, out=out, status=status, max_bytes=cap)
            torch.cuda.synchronize()
        stages = {}
        for ev in prof.key_averages():
            if "jpeg" in ev.key or "Memset" in ev.key:
                stages[ev.key[:60]] = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0)) / 10.0
        res["decode_" + name]["stages_us"] = stages

    # H2D: the compressed bytes of a frame vs the uint8 band of six frames, both from pinned memory
    band_host = torch.empty(plan.band_bytes(n), dtype=torch.uint8).pin_memory()
    band_dev = torch.empty_like(band_host, device=dev)
    for name, src, dst in (("compressed", staged[0][0], data_dev[:staged[0][0].numel()]), ("band", band_host, band_dev)):
        times = []
        for _ in range(20):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dst.copy_(src, non_blocking=True)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        res["h2d_" + name] = dict(bytes=int(src.numel()), median_us=float(np.median(times)) * 1e3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
