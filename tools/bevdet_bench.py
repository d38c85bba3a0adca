#!/usr/bin/env python
"""tools/bevdet_bench.py — BEVDet from the depth net's output to boxes (bevdet.BEVDetHotPath) on an H100.

  python tools/bevdet_bench.py [--steps K] [--warmup W] [--in-flight L] [--no-cpu-check] [--dump-outputs DIR]
  python tools/bevdet_bench.py --temporal [--steps K] [--warmup W] [--in-flight L] [--rounds R] [--no-cpu-check]
  python tools/bevdet_bench.py --temporal --images | --raw-images [--steps K] [--warmup W] [--in-flight L] [--rounds R]
  python tools/bevdet_bench.py --jpeg [--temporal] [--steps K] [--warmup W] [--in-flight L] [--rounds R]
  python tools/bevdet_bench.py --bevdet-nms [--temporal] [--steps K] [--warmup W] [--in-flight L] [--rounds R]

A frame = six cameras of 16 x 44 features (D = 118, C = 80) -> LSS view transform into the 128 x 128 x 96 pixel fp16-pair
image -> CustomResNet + FPN_LSS -> CenterHead (6 tasks) -> centerpoint postprocess -> one D2H.  Reports frames/s with
--in-flight lanes and one frame at a time, for full frames (a new calibration every frame) and for accelerate=True (a
fixed rig: ranks kept); graph-timed stages (pool, encoder, head, postprocess); the dense part's algorithmic GFLOP and
TFLOP/s; the frame graph's node counts; the card name and power limit read in the same run; and a frame-0 check
against the CPU arm (oracle.bevdet.CpuBEVDet).  Prints one JSON line.  Seeded weights, calibrated so that ~1.4 % of
the heat-map cells pass the score threshold: a synthetic workload, not a trained model.

--temporal: BEVDet4D in sequential mode (bevdet.BEVDet4DHotPath) instead: the lanes run independent drives (a fixed rig
on an ego moving 5 m and 0.15 rad per 0.5 s frame, synth.ego_poses), each starting its sequence on its first frame.
Reports frames/s in flight and one at a time for full frames and accelerate=True, measured in rounds that alternate
with the single-frame BEVDet on the same inputs (median of the rounds); the shift graph-timed with its algorithmic bytes
and GB/s; pre_process and the encoder graph-timed with TFLOP/s; the node counts of the start and continue graphs; the
card; and a frame-0 check against the CPU arm (bevdet4d_oracle.CpuBEVDet4D, test infrastructure under tests/).

--images [--bevdet-nms]: BEVDet from six normalised 256 x 704 camera images (bevdet.BEVDetImageHotPath: ResNet-50 stem
kernel, Bottlenecks, CustomFPN and the depth net inside the captured frame; with --bevdet-nms CONFIG_IMG_BEVDET_NMS) next to
the frame from the depth net's output on the same weights and that frame's own depth-net output, measured in rounds that
alternate the two (median of the rounds): frames/s in flight and one at a time; graph-timed stem, layer1-4, neck and
depth net + lss_depth_feat_h16 with their GFLOP and TFLOP/s; the stem's algorithmic bytes and GB/s; the node counts of
both frame graphs; the card; and a frame-0 check against the CPU arm (bevdet_images_oracle.CpuBEVDetImages, tests/).

--raw-images: BEVDet from six decoded 900 x 1600 uint8 camera frames (bevdet.BEVDetFrameHotPath: the test pipeline's
resize, crop and normalisation in p3d_image_prep_u8 at the head of the captured frame) fed from pinned host memory, the
band's H2D included, next to BEVDetImageHotPath on resident fp32 images, in rounds that alternate the two (median of the
rounds): frames/s in flight and one at a time; the host baseline (Pillow + OpenCV prep of the six cameras, one thread,
timed on this host); the graph-timed prep kernel with its algorithmic bytes and GB/s; the band's H2D bytes and time; the
node counts of both frame graphs; the card; and a frame-0 check that the device images equal the host pipeline's.

--temporal --images: BEVDet4D from six normalised 256 x 704 camera images (bevdet.BEVDet4DImageHotPath: the image encoder
and lss_depth_feat_h16 at the head of both the start and the continue graph) next to BEVDet4DHotPath fed that frame's own
depth-net output (merged fp32 logits / tran_feat), in rounds that alternate the two (median of the rounds): frames/s with
--in-flight lanes on independent drives and one at a time; the node counts of the start and continue graphs; the device
memory reserved per lane by its buffers and by capture(); the card; and a frame-0 check against the CPU arm
(bevdet_images_oracle.CpuBEVDetImages.image_encoder -> bevdet4d_oracle.CpuBEVDet4D, tests/).

--temporal --raw-images: BEVDet4D from six decoded 900 x 1600 uint8 camera frames (bevdet.BEVDet4DFrameHotPath) fed from
pinned host memory, the band's H2D included, next to BEVDet4DImageHotPath on resident fp32 images (frames/s in flight and
one at a time); infer_stream over one drive of --steps key frames next to a loop of launch_frames + result over the same
items (frames/s); the node counts of the start and continue graphs; memory per lane; the band's H2D bytes and time; the
card.  Rounds alternate the arms (median of the rounds).

--jpeg [--temporal]: BEVDet (BEVDet4D) from the bytes of six 900 x 1600 JPEG camera files (bevdet.BEVDetJpegHotPath,
BEVDet4DJpegHotPath: the device JPEG decode of the prep plan's band at the head of the captured frame), Pillow-encoded at
q95 4:2:0 by synth.camera_jpegs, the bytes' H2D included, next to the --raw-images arm (BEVDetFrameHotPath /
BEVDet4DFrameHotPath) on Pillow's decode of the same files in pinned memory, in rounds that alternate the two (median):
frames/s in flight and one at a time; the decode of the band, graph-timed (us, compressed MB/s, output GB/s); the H2D
bytes and time per frame of both arms; the host baseline (Pillow's decode of the six files on one thread and on every
core); the node counts of the frame graphs; the card; and a frame-0 check that the lane's band equals Pillow's rows.

--bevdet-nms: the frames with BEVDet's own box decode (bevdet.CONFIG_BEVDET_NMS, with --temporal CONFIG_4D_BEVDET_NMS:
top-K over class x cell, per-class scale-NMS / circle NMS) next to the same weights with the default decode
(centerpoint_postprocess), measured in rounds that alternate the two on the same inputs (median of the rounds): frames/s
in flight and one at a time, both decodes graph-timed on the same head planes in us, the node counts of both frame
graphs, the boxes of frame 0 under each, and the card.
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

from bench import graph_time_ms  # noqa: E402
from pointpillars_bench import gpu_identity  # noqa: E402

BN_GAIN = 6.0 ** 0.5


def _rate(launch, sync, n):
    """frames/s of n calls of launch(i), host clock around work that ends in a device synchronise."""
    sync()
    t0 = time.perf_counter()
    for i in range(n):
        launch(i)
    sync()
    return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--in-flight", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-cpu-check", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the boxes / scores / labels of frame 0 to DIR/*.npy")
    ap.add_argument("--temporal", action="store_true", help="BEVDet4D sequential frames, alternated with BEVDet")
    ap.add_argument("--rounds", type=int, default=3, help="--temporal / --bevdet-nms: alternating measurement rounds")
    ap.add_argument("--bevdet-nms", action="store_true",
                    help="BEVDet's own box decode (scale-NMS / circle NMS), alternated with the default decode")
    ap.add_argument("--images", action="store_true",
                    help="BEVDet from six camera images (ResNet-50 + CustomFPN + depth net in the frame), alternated with "
                         "the frame from the depth net's output")
    ap.add_argument("--raw-images", action="store_true",
                    help="BEVDet from six decoded uint8 camera frames (image prep in the frame), alternated with the frame "
                         "from normalised images")
    ap.add_argument("--jpeg", action="store_true",
                    help="BEVDet (with --temporal BEVDet4D) from the bytes of six JPEG files (device decode in the frame), "
                         "alternated with the frame from Pillow's decode of the same files")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bevdet_bench.py needs a CUDA device (no CPU fallback exists)")
    if args.jpeg:
        return jpeg_files(args)
    if args.temporal and (args.images or args.raw_images):
        return temporal_images(args)
    if args.raw_images:
        return raw_images(args)
    if args.images:
        return images(args)
    if args.bevdet_nms:
        return bevdet_nms(args)
    if args.temporal:
        return temporal(args)
    from paddle3d_b200 import synth
    from paddle3d_b200.bevdet import BEVDet, BEVDetHotPath
    from paddle3d_b200.ops import bev_pool_v2 as bp
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    m = BEVDet(device=dev).init_weight(seed=args.seed, bn_gain=BN_GAIN)
    rigs = [synth.camera_rig(s) for s in range(4)]
    mats = [synth.lss_mats(r) for r in rigs]
    rng = np.random.default_rng(args.seed)
    vt = m.vt
    logits_np = rng.normal(0, 2, (m.N, vt.D, vt.H, vt.W)).astype(np.float32)
    tran_np = rng.normal(0, 1, (m.N, vt.out_channels, vt.H, vt.W)).astype(np.float32)
    logits, tran = torch.from_numpy(logits_np).to(dev), torch.from_numpy(tran_np).to(dev)
    m.calibrate_heatmap_bias(mats[0], logits, tran)
    fl = m.flops()
    line = {"metric": "BEVDet frames/s (6 cams 16x44x118 C=80 -> 128x128 BEV -> CustomResNet + FPN_LSS -> CenterHead -> "
                      "boxes), from the depth net's output", "unit": "frames/s", "gpu": gpu_identity(0),
            "steps": args.steps, "warmup": args.warmup,
            "dense_gflop": {k: v / 1e9 for k, v in fl.items()}}
    lanes_n = max(1, args.in_flight)
    acc_model = BEVDet(accelerate=True, device=dev)
    acc_model.encoder, acc_model.head = m.encoder, m.head
    for acc, model in ((False, m), (True, acc_model)):
        lanes = [BEVDetHotPath(model, device=dev).capture(count_nodes=(i == 0)) for i in range(lanes_n)]
        for ln in lanes:  # inputs written once: the timed frames replay on resident depth-net outputs
            ln.logits.copy_(logits)
            ln.tran_feat.copy_(tran)
        torch.cuda.synchronize()
        pick = (lambda i: mats[i % 4]) if not acc else (lambda i: mats[0])
        for i in range(args.warmup):
            lanes[i % lanes_n].launch(pick(i))
        torch.cuda.synchronize()

        def in_flight(i):
            lanes[i % lanes_n].launch(pick(i))
        r = {"fps_in_flight": _rate(in_flight, torch.cuda.synchronize, args.steps),
             "fps_one_at_a_time": _rate(lambda i: lanes[0].infer(pick(i)), torch.cuda.synchronize, args.steps),
             "lanes": lanes_n}
        for ln in lanes:
            ln.result()  # raises on an fp16-range overflow
        if not acc:
            r["graph_nodes"] = lanes[0].graph_nodes
            got = [t.clone().numpy() for t in lanes[0].infer(mats[0])]
            line["boxes_frame0"] = int(len(got[0]))
        line["accelerate" if acc else "full"] = r
    # graph-timed stages on one stream, on frame 0's ranks
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        prepared = vt._prepare(vt.descriptor(*mats[0]), 1, m.N)
        depth, feat = bp.lss_depth_feat(logits, tran)
        img = m.pool(depth, feat, prepared)
        enc, eshape = m.encode(img)
        h = m.dense(img)
        st.synchronize()

    def head_only():
        s, shape = m.head.shared(enc, eshape)[0], (1, eshape[1], eshape[2], m.head.shared.cout)
        bpar = m.head._batched_params(dev)
        return m.head._tap_sum(m.head._heads_conv_p(s, shape, bpar, dev), bpar, dev)
    t = {"softmax_permute (p3d_lss_depth_feat)": graph_time_ms(lambda: bp.lss_depth_feat(logits, tran, depth, feat), st, 20),
         "pool (memset + p3d_bev_pool_v2_dev_h16)": graph_time_ms(lambda: m.pool(depth, feat, prepared, out=img), st, 20),
         "encoder (CustomResNet + FPN_LSS)": graph_time_ms(lambda: m.encode(img), st, 10),
         "head (shared conv + fused ConvModules / output convs)": graph_time_ms(head_only, st, 10),
         "postprocess (centerpoint_postprocess_device)": graph_time_ms(lambda: m.postprocess(h), st, 10)}
    dense_ms = t["encoder (CustomResNet + FPN_LSS)"] + t["head (shared conv + fused ConvModules / output convs)"]
    line["stages_ms"] = t
    line["dense_tflops"] = {"encoder": (fl["backbone"] + fl["fpn"]) / (t["encoder (CustomResNet + FPN_LSS)"] * 1e-3) / 1e12,
                            "head": fl["head"] / (t["head (shared conv + fused ConvModules / output convs)"] * 1e-3) / 1e12,
                            "dense": fl["total"] / (dense_ms * 1e-3) / 1e12,
                            "note": "algorithmic flops (2 x MACs, Cin 80 unpadded) over graph-timed device time"}
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name, a in zip(("boxes", "scores", "labels"), got):
            np.save(os.path.join(args.dump_outputs, name + ".npy"), a)
    if not args.no_cpu_check:
        from oracle.bevdet import CpuBEVDet
        cams = bp.unpack_cameras(bp.pack_cameras(*mats[0]), 1, m.N)
        axes = tuple(a.numpy() for a in vt.axes_host)
        t0 = time.perf_counter()
        cpu = CpuBEVDet(m.export_numpy(), m.test_cfg, m.label_off).run(cams, axes, logits_np, tran_np, *vt.grid_args())
        s = time.perf_counter() - t0
        paired = 0
        for i in range(len(cpu["boxes"])):
            if not len(got[0]):
                break
            j = int(np.argmin(np.abs(got[0][:, :3] - cpu["boxes"][i, :3]).max(1)))
            e = (np.abs(got[0][j] - cpu["boxes"][i]) / np.maximum(1.0, np.abs(cpu["boxes"][i]))).max()
            paired += int(e <= 1e-3 and got[2][j] == cpu["labels"][i])
        line["cpu_check_frame0"] = {"gpu_boxes": int(len(got[0])), "cpu_boxes": int(len(cpu["boxes"])),
                                    "paired_frac": paired / max(1, len(cpu["boxes"])), "cpu_oracle_s": s,
                                    "kind": "fp64-accumulating numpy + OpenMP oracle, not a tuned CPU implementation"}
    line["value"] = line["full"]["fps_in_flight"]
    print(json.dumps(line))


def temporal(args):
    import torch
    from paddle3d_b200 import synth
    from paddle3d_b200.bevdet import BEVDet, BEVDet4D, BEVDet4DHotPath, BEVDetHotPath
    from paddle3d_b200.frame import copy_rows
    from paddle3d_b200.ops import bev_pool_v2 as bp
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    m4 = BEVDet4D(device=dev).init_weight(seed=args.seed, bn_gain=BN_GAIN)
    m1 = BEVDet(device=dev).init_weight(seed=args.seed, bn_gain=BN_GAIN)
    rigs = [synth.camera_rig(s) for s in range(4)]
    mats = [synth.lss_mats(r) for r in rigs]
    poses = [np.broadcast_to(p, (1, m4.N, 4, 4)) for p in synth.ego_poses(2)]
    prev = [bp.sensor2keyegos(r["sensor2ego"], poses[0], poses[1]) for r in rigs]  # constant motion: one step
    rng = np.random.default_rng(args.seed)
    vt = m4.vt
    logits_np = rng.normal(0, 2, (m4.N, vt.D, vt.H, vt.W)).astype(np.float32)
    tran_np = rng.normal(0, 1, (m4.N, vt.out_channels, vt.H, vt.W)).astype(np.float32)
    logits, tran = torch.from_numpy(logits_np).to(dev), torch.from_numpy(tran_np).to(dev)
    m4.calibrate_heatmap_bias(mats[0], logits, tran)
    m1.calibrate_heatmap_bias(mats[0], logits, tran)
    fl, fl1 = m4.flops(), m1.flops()
    line = {"metric": "BEVDet4D sequential frames/s (6 cams 16x44x118 C=80 -> 128x128 BEV -> pre_process + shift of the "
                      "previous BEV -> CustomResNet(160) + FPN_LSS -> CenterHead -> boxes), from the depth net's output",
            "unit": "frames/s", "gpu": gpu_identity(0), "steps": args.steps, "warmup": args.warmup,
            "dense_gflop": {k: v / 1e9 for k, v in fl.items()}, "bevdet_dense_gflop": fl1["total"] / 1e9}
    lanes_n = max(1, args.in_flight)
    acc4, acc1 = BEVDet4D(accelerate=True, device=dev), BEVDet(accelerate=True, device=dev)
    acc4.encoder, acc4.head, acc4.pre_process = m4.encoder, m4.head, m4.pre_process
    acc1.encoder, acc1.head = m1.encoder, m1.head
    runs = {}
    for name, model, cls in (("bevdet4d_full", m4, BEVDet4DHotPath), ("bevdet_full", m1, BEVDetHotPath),
                             ("bevdet4d_accelerate", acc4, BEVDet4DHotPath), ("bevdet_accelerate", acc1, BEVDetHotPath)):
        lanes = [cls(model, device=dev).capture(count_nodes=(i == 0)) for i in range(lanes_n)]
        for ln in lanes:  # inputs written once: the timed frames replay on resident depth-net outputs
            ln.logits.copy_(logits)
            ln.tran_feat.copy_(tran)
        runs[name] = lanes
    torch.cuda.synchronize()
    frames = {}  # lane -> frames launched (its drive's position)

    def launch(name, lane_i, lane, acc):
        r = lane_i % 4 if not acc else 0  # accelerate: a fixed rig per lane (ranks kept), full: a new calibration
        if "4d" in name:
            k = frames.get((name, lane_i), 0)
            lane.launch(mats[r], prev[r], new_sequence=k == 0)
            frames[(name, lane_i)] = k + 1
        else:
            n = frames.get((name, "n"), 0)
            lane.launch(mats[(lane_i + n) % 4] if not acc else mats[0])
            frames[(name, "n")] = n + 1

    def one_at_a_time(name, lane, acc):
        launch(name, 0, lane, acc)
        lane.result()
    rates = {n: {"fps_in_flight": [], "fps_one_at_a_time": []} for n in runs}
    for name, lanes in runs.items():
        for i in range(args.warmup):
            launch(name, i % lanes_n, lanes[i % lanes_n], "accelerate" in name)
    torch.cuda.synchronize()
    for _ in range(max(1, args.rounds)):  # alternate the models so that clocks and temperature drift hit both
        for name, lanes in runs.items():
            acc = "accelerate" in name
            rates[name]["fps_in_flight"].append(
                _rate(lambda i: launch(name, i % lanes_n, lanes[i % lanes_n], acc), torch.cuda.synchronize, args.steps))
            rates[name]["fps_one_at_a_time"].append(
                _rate(lambda i: one_at_a_time(name, lanes[0], acc), torch.cuda.synchronize, args.steps))
    for name, lanes in runs.items():
        for ln in lanes:
            ln.result()  # raises on an fp16-range overflow
        r = {k: float(np.median(v)) for k, v in rates[name].items()}
        r.update(rounds={k: v for k, v in rates[name].items()}, lanes=lanes_n, graph_nodes=lanes[0].graph_nodes)
        line[name] = r
    line["note_lanes"] = "BEVDet4D lanes run independent drives (each owns its history); frames of one drive are serial"
    # graph-timed stages on one stream, on frame 0's ranks
    st = torch.cuda.Stream(dev)
    hot = runs["bevdet4d_full"][0]
    with torch.cuda.stream(st):
        prepared = vt._prepare(vt.descriptor(*mats[0]), 1, m4.N)
        depth, feat = bp.lss_depth_feat(logits, tran)
        img = m4.pool(depth, feat, prepared)
        _, Y, X, ec = m4.enc_shape
        concat = torch.empty((Y * X, 2 * ec), dtype=torch.float16, device=dev)
        bufs = m4.pre_buffers()
        m4.pre(img, concat, bufs)
        tf = torch.from_numpy(m4.shift_desc(mats[0], prev[0])).to(dev)
        history = hot.history.clone()
        st.synchronize()
    t = {"pre_process (5 convs 80 -> 80, residual epilogue)": graph_time_ms(lambda: m4.pre(img, concat, bufs), st, 10),
         "shift (p3d_bev_shift_h16)": graph_time_ms(lambda: m4.shift(history, tf, concat), st, 50),
         "history copy (2-D memcpy)": graph_time_ms(lambda: copy_rows(history, concat, 384), st, 50),
         "encoder (CustomResNet(160) + FPN_LSS)": graph_time_ms(lambda: m4.encode(concat), st, 10)}
    line["stages_ms"] = t
    shift_bytes = 2 * 4 * m4.bev_C * Y * X
    sms = t["shift (p3d_bev_shift_h16)"]
    line["shift"] = {"algorithmic_bytes": shift_bytes, "GB_per_s": shift_bytes / (sms * 1e-3) / 1e9,
                     "note": "4 C h w read + 4 C h w written (C = 80, 128 x 128); taps re-read from L2"}
    line["dense_tflops"] = {
        "pre_process": fl["pre_process"] / (t["pre_process (5 convs 80 -> 80, residual epilogue)"] * 1e-3) / 1e12,
        "encoder": (fl["backbone"] + fl["fpn"]) / (t["encoder (CustomResNet(160) + FPN_LSS)"] * 1e-3) / 1e12,
        "note": "algorithmic flops (2 x MACs, Cin 80 unpadded) over graph-timed device time"}
    got = [x.clone().numpy() for x in hot.infer(mats[0], None, logits, tran, new_sequence=True)]
    line["boxes_frame0"] = int(len(got[0]))
    if not args.no_cpu_check:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from bevdet4d_oracle import CpuBEVDet4D
        cams = bp.unpack_cameras(bp.pack_cameras(*mats[0]), 1, m4.N)
        axes = tuple(a.numpy() for a in vt.axes_host)
        t0 = time.perf_counter()
        cpu = CpuBEVDet4D(m4.export_numpy(), m4.test_cfg, m4.label_off).run(
            cams, axes, logits_np, tran_np, *vt.grid_args(), rigs[0]["sensor2ego"].astype(np.float64),
            rigs[0]["bda"].astype(np.float64), new_sequence=True)
        s = time.perf_counter() - t0
        paired = 0
        for i in range(len(cpu["boxes"])):
            if not len(got[0]):
                break
            j = int(np.argmin(np.abs(got[0][:, :3] - cpu["boxes"][i, :3]).max(1)))
            e = (np.abs(got[0][j] - cpu["boxes"][i]) / np.maximum(1.0, np.abs(cpu["boxes"][i]))).max()
            paired += int(e <= 1e-3 and got[2][j] == cpu["labels"][i])
        line["cpu_check_frame0"] = {"gpu_boxes": int(len(got[0])), "cpu_boxes": int(len(cpu["boxes"])),
                                    "paired_frac": paired / max(1, len(cpu["boxes"])), "cpu_oracle_s": s,
                                    "kind": "fp64-accumulating numpy + OpenMP oracle, not a tuned CPU implementation"}
    line["value"] = line["bevdet4d_full"]["fps_in_flight"]
    print(json.dumps(line))


def images(args):
    import torch
    from paddle3d_b200 import bevdet as bd
    from paddle3d_b200 import synth
    from paddle3d_b200.ops import bev_pool_v2 as bp
    from paddle3d_b200.ops import dense_conv as dc
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = bd.CONFIG_IMG_BEVDET_NMS if args.bevdet_nms else bd.CONFIG_IMG
    mi = bd.BEVDetFromImages(cfg, device=dev).init_weight(seed=args.seed, bn_gain=BN_GAIN)
    md = bd.BEVDet(dict(cfg), device=dev)  # the frame from the depth net's output, on the same weights
    md.encoder, md.head = mi.encoder, mi.head
    rigs = [synth.camera_rig(s) for s in range(4)]
    mats = [synth.lss_mats(r) for r in rigs]
    imgs_np = synth.camera_images(args.seed)
    imgs = torch.from_numpy(imgs_np).to(dev)
    mi.calibrate_heatmap_bias(mats[0], imgs)
    enc = mi.image_encoder
    vt = mi.vt
    rows, rshape = enc(imgs)
    d = dc.pixel_h16_to_nchw(rows, rshape)
    logits, tran = d[:, :vt.D].contiguous(), d[:, vt.D:vt.D + vt.out_channels].contiguous()
    fl = mi.flops()
    line = {"metric": "BEVDet frames/s from six 256 x 704 camera images (ResNet-50 + CustomFPN + depth net -> LSS -> 128 x "
                      "128 BEV -> CustomResNet + FPN_LSS -> CenterHead -> boxes)", "unit": "frames/s",
            "gpu": gpu_identity(0), "steps": args.steps, "warmup": args.warmup,
            "decode": "bevdet_nms" if args.bevdet_nms else "default", "gflop": {k: v / 1e9 for k, v in fl.items()}}
    lanes_n = max(1, args.in_flight)
    runs = {"images": [bd.BEVDetImageHotPath(mi, device=dev).capture(count_nodes=(i == 0)) for i in range(lanes_n)],
            "depth_net_output": [bd.BEVDetHotPath(md, device=dev).capture(count_nodes=(i == 0)) for i in range(lanes_n)]}
    for ln in runs["images"]:  # inputs written once: the timed frames replay on resident inputs
        ln.imgs.copy_(imgs)
    for ln in runs["depth_net_output"]:
        ln.logits.copy_(logits)
        ln.tran_feat.copy_(tran)
    torch.cuda.synchronize()
    count = {}

    def launch(name, lane):
        k = count.get(name, 0)
        count[name] = k + 1
        lane.launch(mats[k % 4])  # a new calibration every frame
    rates = {n: {"fps_in_flight": [], "fps_one_at_a_time": []} for n in runs}
    for name, lanes in runs.items():
        for i in range(args.warmup):
            launch(name, lanes[i % lanes_n])
    torch.cuda.synchronize()

    def one(name, lane):
        launch(name, lane)
        lane.result()
    for _ in range(max(1, args.rounds)):  # alternate the frames so that clocks and temperature drift hit both
        for name, lanes in runs.items():
            rates[name]["fps_in_flight"].append(
                _rate(lambda i: launch(name, lanes[i % lanes_n]), torch.cuda.synchronize, args.steps))
            rates[name]["fps_one_at_a_time"].append(
                _rate(lambda i: one(name, lanes[0]), torch.cuda.synchronize, args.steps))
    for name, lanes in runs.items():
        for ln in lanes:
            ln.result()  # raises on an fp16-range overflow
        r = {k: float(np.median(v)) for k, v in rates[name].items()}
        r.update(rounds=rates[name], lanes=lanes_n, graph_nodes=lanes[0].graph_nodes)
        line[name] = r
    got = [t.clone().numpy() for t in runs["images"][0].infer(mats[0])]
    line["boxes_frame0"] = int(len(got[0]))
    # graph-timed stages of the image encoder on one stream
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        x0, s0 = enc.stem_forward(imgs)
        ins, x, s = [], x0, s0
        for si in range(len(enc.stages)):
            ins.append((x, s))
            x, s = enc.stage_forward(si, x, s)
        feats = enc.backbone(imgs)
        y, ys = enc.neck(feats)
        depth, feat = mi.depth_feat(rows, rshape)
        st.synchronize()
    t = {"stem": graph_time_ms(lambda: enc.stem_forward(imgs), st, 20)}
    for si in range(len(enc.stages)):
        t["layer%d" % (si + 1)] = graph_time_ms(lambda: enc.stage_forward(si, *ins[si]), st, 10)
    t["neck"] = graph_time_ms(lambda: enc.neck(feats), st, 10)
    t["depth_net + lss_depth_feat_h16"] = graph_time_ms(lambda: mi.depth_feat(*enc.head(y, ys), depth, feat), st, 20)
    t["image_encoder (all of the above but lss_depth_feat_h16)"] = graph_time_ms(lambda: enc(imgs), st, 5)
    H, W = mi.input_size
    n = mi.N
    gf = {"stem": fl["img_stem"]}
    h, w = dc.stem_shape(H, W)
    for si, stage in enumerate(enc.stages):
        sub = 0.0
        for blk in stage:
            s_ = blk["conv2"].stride
            oh, ow = (h - 1) // s_ + 1, (w - 1) // s_ + 1
            sub += 2.0 * n * (h * w * blk["conv1"].cin * blk["conv1"].cout + oh * ow * 9 * blk["conv2"].cin * blk["conv2"].cout
                              + oh * ow * blk["conv3"].cin * blk["conv3"].cout)
            if blk["down"] is not None:
                sub += 2.0 * n * oh * ow * blk["down"].cin * blk["down"].cout
            h, w = oh, ow
        gf["layer%d" % (si + 1)] = sub
    gf["neck"] = fl["img_neck"]
    gf["depth_net + lss_depth_feat_h16"] = fl["depth_net"]
    gf["image_encoder (all of the above but lss_depth_feat_h16)"] = fl["img_total"]
    line["stages"] = {k: {"ms": t[k], "gflop": gf[k] / 1e9, "tflops": gf[k] / (t[k] * 1e-3) / 1e12} for k in t}
    ph, pw = dc.stem_shape(H, W)
    stem_bytes = n * 3 * H * W * 4 + n * ph * pw * 64 * 4
    line["stem_bytes"] = {"algorithmic_bytes": stem_bytes, "GB_per_s": stem_bytes / (t["stem"] * 1e-3) / 1e9,
                          "note": "fp32 images read once + pixel fp16-pair rows written once"}
    line["note"] = "algorithmic flops (2 x MACs; the depth net's 198 outputs unpadded) over graph-timed device time"
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name, a in zip(("boxes", "scores", "labels"), got):
            np.save(os.path.join(args.dump_outputs, name + ".npy"), a)
    if not args.no_cpu_check:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from bevdet_images_oracle import CpuBEVDetImages
        cams = bp.unpack_cameras(bp.pack_cameras(*mats[0]), 1, mi.N)
        axes = tuple(a.numpy() for a in vt.axes_host)
        t0 = time.perf_counter()
        cpu = CpuBEVDetImages(mi.export_numpy(), mi.test_cfg, mi.label_off).run(cams, axes, imgs_np, *vt.grid_args())
        s = time.perf_counter() - t0
        if args.bevdet_nms:
            from bevdet_postprocess_oracle import bevdet_postprocess_ref
            cpu["boxes"], cpu["scores"], cpu["labels"], _ = bevdet_postprocess_ref(cpu["head"], mi.test_cfg, mi.label_off)
        paired = 0
        for i in range(len(cpu["boxes"])):
            if not len(got[0]):
                break
            j = int(np.argmin(np.abs(got[0][:, :3] - cpu["boxes"][i, :3]).max(1)))
            e = (np.abs(got[0][j] - cpu["boxes"][i]) / np.maximum(1.0, np.abs(cpu["boxes"][i]))).max()
            paired += int(e <= 1e-3 and got[2][j] == cpu["labels"][i])
        gl = d.cpu().numpy()
        err = float(np.abs(gl[:, :vt.D] - cpu["logits"]).max() / np.abs(cpu["logits"]).max())
        line["cpu_check_frame0"] = {"gpu_boxes": int(len(got[0])), "cpu_boxes": int(len(cpu["boxes"])),
                                    "paired_frac": paired / max(1, len(cpu["boxes"])), "logits_max_abs_over_max": err,
                                    "cpu_oracle_s": s,
                                    "kind": "fp64-accumulating numpy + OpenMP oracle, not a tuned CPU implementation"}
    line["value"] = line["images"]["fps_in_flight"]
    print(json.dumps(line))


def raw_images(args):
    import cv2
    import torch
    from paddle3d_b200 import bevdet as bd
    from paddle3d_b200 import synth
    from paddle3d_b200.ops import image_prep as ip
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from image_prep_oracle import pipeline_pil_cv2
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    m = bd.BEVDetFromImages(device=dev).init_weight(seed=args.seed, bn_gain=BN_GAIN)
    plan, dcfg, aug = m.prep_plan, m.data_config, m.augmentation
    rigs = [synth.camera_rig(s) for s in range(4)]
    cams = [(r["sensor2ego"], r["cam2imgs"], r["bda"]) for r in rigs]
    mats = [m.test_mats(*c) for c in cams]
    frames_np = [synth.camera_frames(args.seed + i) for i in range(2)]
    frames_host = [torch.from_numpy(f).pin_memory() for f in frames_np]
    imgs = ip.image_prep_u8(frames_host[0].to(dev), plan)
    m.calibrate_heatmap_bias(mats[0], imgs)
    line = {"metric": "BEVDet frames/s from six decoded 900 x 1600 uint8 camera frames in pinned host memory (band H2D -> "
                      "resize / crop / normalise -> ResNet-50 + CustomFPN + depth net -> LSS -> BEV encoder -> CenterHead "
                      "-> boxes)", "unit": "frames/s", "gpu": gpu_identity(0), "steps": args.steps,
            "warmup": args.warmup}
    lanes_n = max(1, args.in_flight)
    runs = {"frames": [bd.BEVDetFrameHotPath(m, device=dev).capture(count_nodes=(i == 0)) for i in range(lanes_n)],
            "images": [bd.BEVDetImageHotPath(m, device=dev).capture(count_nodes=(i == 0)) for i in range(lanes_n)]}
    for ln in runs["images"]:  # resident fp32 images: the timed frames replay on them
        ln.imgs.copy_(imgs)
    torch.cuda.synchronize()
    count = {}

    def launch(name, lane):
        k = count.get(name, 0)
        count[name] = k + 1
        if name == "frames":  # a new calibration and new frames every frame
            lane.launch_frames(*cams[k % 4], frames_host[k % 2])
        else:
            lane.launch(mats[k % 4])

    def one(name, lane):
        launch(name, lane)
        lane.result()
    rates = {n: {"fps_in_flight": [], "fps_one_at_a_time": []} for n in runs}
    for name, lanes in runs.items():
        for i in range(args.warmup):
            launch(name, lanes[i % lanes_n])
    torch.cuda.synchronize()
    for _ in range(max(1, args.rounds)):  # alternate the frames so that clocks and temperature drift hit both
        for name, lanes in runs.items():
            rates[name]["fps_in_flight"].append(
                _rate(lambda i: launch(name, lanes[i % lanes_n]), torch.cuda.synchronize, args.steps))
            rates[name]["fps_one_at_a_time"].append(
                _rate(lambda i: one(name, lanes[0]), torch.cuda.synchronize, args.steps))
    for name, lanes in runs.items():
        for ln in lanes:
            ln.result()  # raises on an fp16-range overflow
        r = {k: float(np.median(v)) for k, v in rates[name].items()}
        r.update(rounds=rates[name], lanes=lanes_n, graph_nodes=lanes[0].graph_nodes)
        line[name] = r
    hot = runs["frames"][0]
    got = [t.clone().numpy() for t in hot.infer_frames(*cams[0], frames_host[0])]
    line["boxes_frame0"] = int(len(got[0]))
    # host baseline: Pillow resize + crop and mmcv.imnormalize's OpenCV steps of the six cameras, one thread
    cv2.setNumThreads(1)
    reps = 5
    host_imgs = pipeline_pil_cv2(frames_np[0], aug["resize_dims"], aug["crop"], dcfg["mean"], dcfg["std"], dcfg["to_rgb"])
    t0 = time.perf_counter()
    for i in range(reps):
        pipeline_pil_cv2(frames_np[i % 2], aug["resize_dims"], aug["crop"], dcfg["mean"], dcfg["std"], dcfg["to_rgb"])
    host_s = (time.perf_counter() - t0) / reps
    line["host_prep"] = {"s_per_frame": host_s, "frames_per_s": 1.0 / host_s, "cpus": os.cpu_count(),
                         "kind": "PIL.Image.resize + crop and cv2 cvtColor / subtract / multiply of six 900 x 1600 frames, "
                                 "one thread, no H2D"}
    dev_imgs = hot.imgs.cpu().numpy()
    line["images_equal_host_pipeline_frame0"] = bool(np.array_equal(dev_imgs.view(np.int32), host_imgs.view(np.int32)))
    # the prep kernel, graph-timed, and the band's H2D
    st = torch.cuda.Stream(dev)
    band, out = hot.band, torch.empty_like(hot.imgs)
    prep_ms = graph_time_ms(lambda: ip.image_prep_u8(band, plan, out=out), st, 50)
    n = m.N
    nbytes = plan.band_bytes(n) + plan.out_bytes(n)
    line["prep_kernel"] = {"us": prep_ms * 1e3, "algorithmic_bytes": nbytes, "GB_per_s": nbytes / (prep_ms * 1e-3) / 1e9,
                           "band_rows": plan.band_rows,
                           "note": "the band of six cameras read once (uint8) + the fp32 images written once"}
    with torch.cuda.stream(st):
        hot.copy_band(frames_host[0])
        st.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(st)
        for _ in range(20):
            hot.copy_band(frames_host[0])
        e.record(st)
    e.synchronize()
    h2d_ms = s.elapsed_time(e) / 20
    line["band_h2d"] = {"bytes_per_frame": plan.band_bytes(n), "ms": h2d_ms,
                        "GB_per_s": plan.band_bytes(n) / (h2d_ms * 1e-3) / 1e9,
                        "full_fp32_images_bytes": plan.out_bytes(n)}
    line["value"] = line["frames"]["fps_in_flight"]
    print(json.dumps(line))


def jpeg_files(args):
    import io
    from concurrent.futures import ThreadPoolExecutor

    import torch
    from PIL import Image

    from paddle3d_b200 import bevdet as bd
    from paddle3d_b200 import synth
    from paddle3d_b200.frame import count_graph_nodes
    from paddle3d_b200.ops import jpeg
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    four = args.temporal
    m = (bd.BEVDet4DFromImages if four else bd.BEVDetFromImages)(device=dev).init_weight(seed=args.seed, bn_gain=BN_GAIN)
    plan = m.prep_plan
    files = [synth.camera_jpegs(args.seed + i, quality=95, subsampling=2) for i in range(2)]

    def pil(f):
        return np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))
    frames_host = [torch.from_numpy(np.stack([pil(f) for f in fr])).pin_memory() for fr in files]
    L = 8
    if four:
        rig = synth.camera_rig(args.seed, bda=False)
        poses = synth.ego_poses(L, speed=10.0, yaw_rate=0.3)
        items = [(None, rig["sensor2ego"][0], np.broadcast_to(p, (m.N, 4, 4)).copy(), rig["cam2imgs"][0]) for p in poses]
        steps = list(bd.drive_mats(items, m.test_mats))
        m.calibrate_heatmap_bias(steps[0][0], m.images_from_frames(frames_host[0].to(dev)))
    else:
        rigs = [synth.camera_rig(s) for s in range(4)]
        cams = [(r["sensor2ego"], r["cam2imgs"], r["bda"]) for r in rigs]
        m.calibrate_heatmap_bias(m.test_mats(*cams[0]), m.images_from_frames(frames_host[0].to(dev)))
    line = {"metric": "BEVDet%s frames/s from the bytes of six 900 x 1600 JPEG camera files (q95 4:2:0; H2D of the bytes -> "
                      "device JPEG decode of the band -> resize / crop / normalise -> ResNet-50 + CustomFPN + depth net -> "
                      "LSS -> BEV encoder -> CenterHead -> boxes)" % ("4D sequential" if four else ""),
            "unit": "frames/s", "gpu": gpu_identity(0), "steps": args.steps, "warmup": args.warmup,
            "compressed_bytes_per_frame": [sum(len(f) for f in fr) for fr in files]}
    lanes_n = max(1, args.in_flight)
    arms = {"jpeg": bd.BEVDet4DJpegHotPath if four else bd.BEVDetJpegHotPath,
            "frames": bd.BEVDet4DFrameHotPath if four else bd.BEVDetFrameHotPath}
    runs = {n: [c(m, device=dev).capture(count_nodes=(i == 0)) for i in range(lanes_n)] for n, c in arms.items()}
    torch.cuda.synchronize()
    count = {}

    def launch(name, lane_i, lane):
        k = count.get((name, lane_i), 0)
        count[(name, lane_i)] = k + 1
        if four:
            mats, prev, _ = steps[0 if k == 0 else 1 + (k - 1) % (L - 1)]
            args_ = (mats[0], mats[1], mats[4])
            extra = (prev, k == 0)
        else:
            args_, extra = cams[k % 4], ()
        if name == "jpeg":
            lane.launch_jpegs(*args_, files[k % 2], *extra)
        else:
            lane.launch_frames(*args_, frames_host[k % 2], *extra)

    def one(name, lane):
        launch(name, 0, lane)
        lane.result()
    rates = {n: {"fps_in_flight": [], "fps_one_at_a_time": []} for n in runs}
    for name, lanes in runs.items():
        for i in range(args.warmup):
            launch(name, i % lanes_n, lanes[i % lanes_n])
    torch.cuda.synchronize()
    for _ in range(max(1, args.rounds)):  # alternate the arms so that clocks and temperature drift hit both
        for name, lanes in runs.items():
            rates[name]["fps_in_flight"].append(
                _rate(lambda i: launch(name, i % lanes_n, lanes[i % lanes_n]), torch.cuda.synchronize, args.steps))
            rates[name]["fps_one_at_a_time"].append(
                _rate(lambda i: one(name, lanes[0]), torch.cuda.synchronize, args.steps))
    for name, lanes in runs.items():
        for ln in lanes:
            ln.result()  # raises on a JPEG decode error or an fp16-range overflow
        r = {k: float(np.median(v)) for k, v in rates[name].items()}
        r.update(rounds=rates[name], lanes=lanes_n,
                 graph_nodes={g: count_graph_nodes(x) for g, x in lanes[0].graphs.items()} if four else
                 lanes[0].graph_nodes)
        line[name] = r
    hot = runs["jpeg"][0]
    line["band_equals_pillow_frame"] = bool(np.array_equal(hot.band.cpu().numpy(),
                                                           frames_host[(count[("jpeg", 0)] - 1) % 2].numpy()[
                                                               :, plan.band[0]:plan.band[1]]))
    # the decode of the band alone, graph-timed
    st = torch.cuda.Stream(dev)
    nbytes = hot.pack_jpegs(files[0])
    hot.jpeg_data[:nbytes].copy_(hot.h_jpeg_data[:nbytes])
    hot.jpeg_desc.copy_(hot.h_jpeg_desc)
    status = torch.zeros(m.N, dtype=torch.int32, device=dev)
    out = torch.empty_like(hot.band)
    dec_ms = graph_time_ms(lambda: jpeg.jpeg_decode_u8(hot.jpeg_data, hot.jpeg_desc, m.N, plan.src_size, rows=plan.band,
                                                       out=out, status=status, max_bytes=hot.jpeg_max_bytes), st, 50)
    comp = line["compressed_bytes_per_frame"][0]
    line["decode_band"] = {"us": dec_ms * 1e3, "compressed_MB_per_s": comp / (dec_ms * 1e-3) / 1e6,
                           "output_GB_per_s": out.numel() / (dec_ms * 1e-3) / 1e9, "band_rows": plan.band_rows}

    def h2d_ms(copy):
        with torch.cuda.stream(st):
            copy()
            st.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(st)
            for _ in range(20):
                copy()
            e.record(st)
        e.synchronize()
        return s.elapsed_time(e) / 20

    def jpeg_copy():
        hot.jpeg_data[:nbytes].copy_(hot.h_jpeg_data[:nbytes], non_blocking=True)
        hot.jpeg_desc.copy_(hot.h_jpeg_desc, non_blocking=True)
    fh = runs["frames"][0]
    line["h2d"] = {"jpeg": {"bytes_per_frame": nbytes + hot.jpeg_desc.numel(), "ms": h2d_ms(jpeg_copy)},
                   "frames_band": {"bytes_per_frame": plan.band_bytes(m.N),
                                   "ms": h2d_ms(lambda: fh.copy_band(frames_host[0]))}}
    # host baseline: Pillow's decode of the six files, one thread and every core
    reps = 5
    t0 = time.perf_counter()
    for i in range(reps):
        for f in files[i % 2]:
            pil(f)
    one_s = (time.perf_counter() - t0) / reps
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        list(ex.map(pil, files[0]))
        t0 = time.perf_counter()
        for i in range(reps):
            list(ex.map(pil, files[i % 2]))
        all_s = (time.perf_counter() - t0) / reps
    line["host_decode"] = {"one_thread_s_per_frame": one_s, "all_cores_s_per_frame": all_s, "cpus": os.cpu_count(),
                           "kind": "np.asarray(Image.open(f).convert('RGB')) of the six files (libjpeg-turbo)"}
    line["value"] = line["jpeg"]["fps_in_flight"]
    print(json.dumps(line))


def _lanes(make, n):
    """n captured lanes (make() builds one) and the device memory each reserved: by its buffers, then by capture() (its
    graphs' private pools; the first lane's also holds the warm-up's cached blocks, which later lanes reuse)."""
    import torch
    lanes, mem = [], []
    for i in range(n):
        torch.cuda.synchronize()
        r0 = torch.cuda.memory_reserved()
        ln = make()
        r1 = torch.cuda.memory_reserved()
        ln.capture(count_nodes=i == 0)
        torch.cuda.synchronize()
        r2 = torch.cuda.memory_reserved()
        lanes.append(ln)
        mem.append({"buffers_MiB": (r1 - r0) / 2 ** 20, "capture_MiB": (r2 - r1) / 2 ** 20})
    return lanes, mem


def temporal_images(args):
    import torch
    from paddle3d_b200 import bevdet as bd
    from paddle3d_b200 import synth
    from paddle3d_b200.frame import count_graph_nodes
    from paddle3d_b200.ops import bev_pool_v2 as bp
    from paddle3d_b200.ops import dense_conv as dc
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    m = bd.BEVDet4DFromImages(device=dev).init_weight(seed=args.seed, bn_gain=BN_GAIN)
    vt = m.vt
    # one drive of pinned camera frames on a rig turning at 0.15 rad per 0.5 s key frame (drive_mats' matrices); the
    # lanes run it independently, each starting its sequence on its first frame
    rig = synth.camera_rig(args.seed, bda=False)
    L = 8
    frames_host = [torch.from_numpy(synth.camera_frames(args.seed + i)).pin_memory() for i in range(2)]
    items = [(frames_host[k % 2], rig["sensor2ego"][0], np.broadcast_to(p, (m.N, 4, 4)).copy(), rig["cam2imgs"][0])
             for k, p in enumerate(synth.ego_poses(L, speed=10.0, yaw_rate=0.3))]
    steps = list(bd.drive_mats(items, m.test_mats))
    imgs = m.images_from_frames(frames_host[0].to(dev))
    imgs_np = imgs.cpu().numpy()
    m.calibrate_heatmap_bias(steps[0][0], imgs)
    rows, rshape = m.image_encoder(imgs)
    d = dc.pixel_h16_to_nchw(rows, rshape)
    logits, tran = d[:, :vt.D].contiguous(), d[:, vt.D:vt.D + vt.out_channels].contiguous()
    raw = args.raw_images
    src = ("decoded 900 x 1600 uint8 camera frames in pinned host memory (band H2D -> resize / crop / normalise -> "
           if raw else "256 x 704 camera images (")
    line = {"metric": "BEVDet4D sequential frames/s from six " + src + "ResNet-50 + CustomFPN + depth net -> LSS -> "
                      "pre_process + shift of the previous BEV -> CustomResNet(160) + FPN_LSS -> CenterHead -> boxes)",
            "unit": "frames/s", "gpu": gpu_identity(0), "steps": args.steps, "warmup": args.warmup,
            "gflop": {k: v / 1e9 for k, v in m.flops().items()}}
    lanes_n = max(1, args.in_flight)
    if raw:
        arms = {"frames": bd.BEVDet4DFrameHotPath, "images": bd.BEVDet4DImageHotPath}
    else:
        arms = {"images": bd.BEVDet4DImageHotPath, "depth_net_output": bd.BEVDet4DHotPath}
    runs, mem = {}, {}
    for name, cls in arms.items():
        runs[name], mem[name] = _lanes(lambda: cls(m, device=dev), lanes_n)
    for ln in runs["images"]:  # resident inputs: the timed frames replay on them
        ln.imgs.copy_(imgs)
    for ln in runs.get("depth_net_output", []):
        ln.logits.copy_(logits)
        ln.tran_feat.copy_(tran)
    torch.cuda.synchronize()
    count = {}

    def launch(name, lane_i, lane):
        k = count.get((name, lane_i), 0)
        count[(name, lane_i)] = k + 1
        mats, prev, _ = steps[0 if k == 0 else 1 + (k - 1) % (L - 1)]
        if name == "frames":
            it = items[k % L]
            lane.launch_frames(mats[0], mats[1], mats[4], it[0], prev, k == 0)
        elif name == "images":
            lane.launch(mats, prev, None, k == 0)
        else:
            lane.launch(mats, prev, None, None, k == 0)

    def one(name, lane):
        launch(name, 0, lane)
        lane.result()
    rates = {n: {"fps_in_flight": [], "fps_one_at_a_time": []} for n in runs}
    for name, lanes in runs.items():
        for i in range(args.warmup):
            launch(name, i % lanes_n, lanes[i % lanes_n])
    torch.cuda.synchronize()
    if raw:  # one drive of --steps key frames: infer_stream against launch_frames + result per item
        drive = [(frames_host[k % 2], rig["sensor2ego"][0], np.broadcast_to(p, (m.N, 4, 4)).copy(), rig["cam2imgs"][0])
                 for k, p in enumerate(synth.ego_poses(args.steps, speed=10.0, yaw_rate=0.3))]
        plan = list(bd.drive_mats(drive, m.test_mats))
        stream_lane = runs["frames"][0]

        def loop():
            for it, (mats, prev, new) in zip(drive, plan):
                stream_lane.infer_frames(mats[0], mats[1], mats[4], it[0], prev, new)

        def drive_rate(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return len(drive) / (time.perf_counter() - t0)
        rates["drive"] = {"infer_stream": [], "launch_frames_result_loop": []}
        for _ in stream_lane.infer_stream(drive[:args.warmup]):
            pass
    for _ in range(max(1, args.rounds)):  # alternate the arms so that clocks and temperature drift hit both
        for name, lanes in runs.items():
            rates[name]["fps_in_flight"].append(
                _rate(lambda i: launch(name, i % lanes_n, lanes[i % lanes_n]), torch.cuda.synchronize, args.steps))
            rates[name]["fps_one_at_a_time"].append(
                _rate(lambda i: one(name, lanes[0]), torch.cuda.synchronize, args.steps))
        if raw:
            rates["drive"]["infer_stream"].append(drive_rate(lambda: [None for _ in stream_lane.infer_stream(drive)]))
            rates["drive"]["launch_frames_result_loop"].append(drive_rate(loop))
    for name, lanes in runs.items():
        for ln in lanes:
            ln.result()  # raises on an fp16-range overflow
        r = {k: float(np.median(v)) for k, v in rates[name].items()}
        r.update(rounds=rates[name], lanes=lanes_n, memory_reserved_per_lane=mem[name],
                 graph_nodes={g: count_graph_nodes(x) for g, x in lanes[0].graphs.items()})
        line[name] = r
    if raw:
        line["drive"] = dict({k: float(np.median(v)) for k, v in rates["drive"].items()}, rounds=rates["drive"],
                             key_frames=len(drive), note="frames/s of one drive on one lane; frames of a drive are serial")
    line["note_lanes"] = "lanes run independent drives (each owns its history); frames of one drive are serial"
    hot = runs["images"][0]
    got = [t.clone().numpy() for t in hot.infer(steps[0][0], None, imgs, new_sequence=True)]
    line["boxes_frame0"] = int(len(got[0]))
    if raw:
        plan_ = m.prep_plan
        st = torch.cuda.Stream(dev)
        fh = runs["frames"][0]
        with torch.cuda.stream(st):
            fh.copy_band(frames_host[0])
            st.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(st)
            for _ in range(20):
                fh.copy_band(frames_host[0])
            e.record(st)
        e.synchronize()
        h2d_ms = s.elapsed_time(e) / 20
        line["band_h2d"] = {"bytes_per_frame": plan_.band_bytes(m.N), "ms": h2d_ms,
                            "GB_per_s": plan_.band_bytes(m.N) / (h2d_ms * 1e-3) / 1e9}
        line["value"] = line["frames"]["fps_in_flight"]
        print(json.dumps(line))
        return
    if not args.no_cpu_check:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from bevdet4d_oracle import CpuBEVDet4D
        from bevdet_images_oracle import CpuBEVDetImages
        w = m.export_numpy()
        mats = steps[0][0]
        cams = bp.unpack_cameras(bp.pack_cameras(*mats), 1, m.N)
        axes = tuple(a.numpy() for a in vt.axes_host)
        t0 = time.perf_counter()
        cl, ct = CpuBEVDetImages(w, m.test_cfg, m.label_off).image_encoder(imgs_np)
        cpu = CpuBEVDet4D(w, m.test_cfg, m.label_off).run(cams, axes, cl, ct, *vt.grid_args(),
                                                          np.asarray(mats[0], np.float64),
                                                          np.asarray(mats[4], np.float64), new_sequence=True)
        s = time.perf_counter() - t0
        paired = 0
        for i in range(len(cpu["boxes"])):
            if not len(got[0]):
                break
            j = int(np.argmin(np.abs(got[0][:, :3] - cpu["boxes"][i, :3]).max(1)))
            e = (np.abs(got[0][j] - cpu["boxes"][i]) / np.maximum(1.0, np.abs(cpu["boxes"][i]))).max()
            paired += int(e <= 1e-3 and got[2][j] == cpu["labels"][i])
        line["cpu_check_frame0"] = {"gpu_boxes": int(len(got[0])), "cpu_boxes": int(len(cpu["boxes"])),
                                    "paired_frac": paired / max(1, len(cpu["boxes"])), "cpu_oracle_s": s,
                                    "kind": "fp64-accumulating numpy + OpenMP oracle, not a tuned CPU implementation"}
    line["value"] = line["images"]["fps_in_flight"]
    print(json.dumps(line))


def bevdet_nms(args):
    import torch
    from paddle3d_b200 import bevdet as bd
    from paddle3d_b200 import synth
    from paddle3d_b200.ops import bev_pool_v2 as bp
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    four = args.temporal
    model_cls, hot_cls = (bd.BEVDet4D, bd.BEVDet4DHotPath) if four else (bd.BEVDet, bd.BEVDetHotPath)
    cfgs = {"default_decode": bd.CONFIG_4D if four else bd.CONFIG,
            "bevdet_nms": bd.CONFIG_4D_BEVDET_NMS if four else bd.CONFIG_BEVDET_NMS}
    models = {}
    for name, cfg in cfgs.items():  # one set of weights under both test configs
        m = model_cls(cfg, device=dev)
        if models:
            first = models["default_decode"]
            m.encoder, m.head = first.encoder, first.head
            if four:
                m.pre_process = first.pre_process
        else:
            m.init_weight(seed=args.seed, bn_gain=BN_GAIN)
        models[name] = m
    m0 = models["default_decode"]
    rigs = [synth.camera_rig(s) for s in range(4)]
    mats = [synth.lss_mats(r) for r in rigs]
    poses = [np.broadcast_to(p, (1, m0.N, 4, 4)) for p in synth.ego_poses(2)]
    prev = [bp.sensor2keyegos(r["sensor2ego"], poses[0], poses[1]) for r in rigs]
    rng = np.random.default_rng(args.seed)
    vt = m0.vt
    logits = torch.from_numpy(rng.normal(0, 2, (m0.N, vt.D, vt.H, vt.W)).astype(np.float32)).to(dev)
    tran = torch.from_numpy(rng.normal(0, 1, (m0.N, vt.out_channels, vt.H, vt.W)).astype(np.float32)).to(dev)
    m0.calibrate_heatmap_bias(mats[0], logits, tran)
    line = {"metric": "%s frames/s with BEVDet's own box decode (scale-NMS / circle NMS) next to the default decode, from "
                      "the depth net's output" % ("BEVDet4D sequential" if four else "BEVDet"),
            "unit": "frames/s", "gpu": gpu_identity(0), "steps": args.steps, "warmup": args.warmup}
    lanes_n = max(1, args.in_flight)
    runs = {}
    for name, m in models.items():
        lanes = [hot_cls(m, device=dev).capture(count_nodes=(i == 0)) for i in range(lanes_n)]
        for ln in lanes:  # inputs written once: the timed frames replay on resident depth-net outputs
            ln.logits.copy_(logits)
            ln.tran_feat.copy_(tran)
        runs[name] = lanes
    torch.cuda.synchronize()
    frames = {}

    def launch(name, lane_i, lane):
        k = frames.get((name, lane_i), 0)
        frames[(name, lane_i)] = k + 1
        r = (lane_i + k) % 4  # a new calibration every frame
        if four:
            lane.launch(mats[lane_i % 4], prev[lane_i % 4], new_sequence=k == 0)
        else:
            lane.launch(mats[r])

    def one_at_a_time(name, lane):
        launch(name, 0, lane)
        lane.result()
    rates = {n: {"fps_in_flight": [], "fps_one_at_a_time": []} for n in runs}
    for name, lanes in runs.items():
        for i in range(args.warmup):
            launch(name, i % lanes_n, lanes[i % lanes_n])
    torch.cuda.synchronize()
    for _ in range(max(1, args.rounds)):  # alternate the decodes so that clocks and temperature drift hit both
        for name, lanes in runs.items():
            rates[name]["fps_in_flight"].append(
                _rate(lambda i: launch(name, i % lanes_n, lanes[i % lanes_n]), torch.cuda.synchronize, args.steps))
            rates[name]["fps_one_at_a_time"].append(
                _rate(lambda i: one_at_a_time(name, lanes[0]), torch.cuda.synchronize, args.steps))
    # both decodes graph-timed on the same head planes (frame 0)
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        x = m0.encoder_input(mats[0], None, logits, tran) if four else m0.image(mats[0], logits, tran)
        h = m0.dense(x)
        st.synchronize()
    for name, lanes in runs.items():
        for ln in lanes:
            ln.result()  # raises on an fp16-range overflow
        m = models[name]
        r = {k: float(np.median(v)) for k, v in rates[name].items()}
        got = lanes[0].infer(mats[0], None, new_sequence=True) if four else lanes[0].infer(mats[0])
        r.update(rounds=rates[name], lanes=lanes_n, graph_nodes=lanes[0].graph_nodes, boxes_frame0=int(len(got[0])),
                 result_rows=m.result_rows(), decode_us=1e3 * graph_time_ms(lambda: m.postprocess(h), st, 50))
        line[name] = r
    line["value"] = line["bevdet_nms"]["fps_in_flight"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
