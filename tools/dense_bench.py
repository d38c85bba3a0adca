#!/usr/bin/env python
"""Per-layer timing of the dense RPN / neck / CenterHead (SURVEY §8f-1) at the C3 shapes (BEV [1, 256, 180, 180]).

Graph-replayed, one JSON line per distinct layer shape and kernel variant with its algorithmic TFLOP/s (2 * MACs of the
convolution; the kernels execute 3 fp16 MMAs per product), then the whole head.  Needs a GPU:
    python tools/dense_bench.py [--variants] [> dense_layers.jsonl]

--trace builds the library with -DP3D_DENSE_TRACE into a temporary directory and prints, per layer, where the dense
kernel's time goes, in SM cycles per work item (summed over the CTAs, divided by the items): the consumer warpgroups'
waits on the activation / weight "full" barriers, in wgmma.wait_group, their epilogue (staging the accumulators) and
their waits for a free staging tile; the producer thread's waits on "empty" barriers; epilogue thread 0's waits on
"staged" and its time from "staged" to "freed" (these layers write only the pixel H16 image: the TMA stores of the
consumers' fp16-pair tile until they have read it).  Cycles are clock64 counts; the trace build is slower than the
default one.
"""
import argparse
import ctypes
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from paddle3d_b200.dense_head import DenseRPNHead, _Conv  # noqa: E402
from paddle3d_b200.ops import dense_conv as dc  # noqa: E402


def graph_time(fn, iters=10):
    st = torch.cuda.current_stream()
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    g.replay()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) / iters * 1e3  # us


SHAPES = [  # (name, cin, cout, k, stride, pad, up, h, w) at the C3 BEV size 180 x 180
    ("backbone0 256->128 s1", 256, 128, 3, 1, 1, 1, 180, 180), ("backbone0 128->128", 128, 128, 3, 1, 1, 1, 180, 180),
    ("backbone1 128->256 s2", 128, 256, 3, 2, 1, 1, 180, 180), ("backbone1 256->256", 256, 256, 3, 1, 1, 1, 90, 90),
    ("neck 1x1 128->256", 128, 256, 1, 1, 0, 1, 180, 180), ("neck deconv 256->256 x2", 256, 256, 2, 2, 0, 2, 90, 90),
    ("shared 512->64", 512, 64, 3, 1, 1, 1, 180, 180), ("heads 64->2304 (36 batched)", 64, 2304, 3, 1, 1, 1, 180, 180),
]
# per-CTA fields of the trace build (dcf::TraceField in csrc/dense_conv_f16.cu)
TRACE_FIELDS = ["items", "cycles", "a_full", "a_full_1", "b_full", "b_full_1", "mma_wait", "mma_wait_1", "epilogue",
                "epilogue_1", "stage_free", "stage_free_1", "prod_a_empty", "prod_b_empty", "epi_warps_wait",
                "epi_warps_busy"]


def trace():
    from paddle3d_b200 import _lib
    from paddle3d_b200 import build as b
    out = tempfile.mkdtemp(prefix="p3d_dense_trace_")
    _lib.LIB_PATH = b.build(out_dir=out, extra_flags=["-DP3D_DENSE_TRACE"])
    rd = _lib.lib().p3d_dense_trace_read
    rd.restype, rd.argtypes = ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    nf = rd(None, 0, 1)
    assert nf == len(TRACE_FIELDS), "trace fields: library %d, tool %d" % (nf, len(TRACE_FIELDS))
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    rng = np.random.default_rng(0)
    max_ctas = 1024
    buf = np.zeros((max_ctas, nf), np.uint64)
    for name, cin, cout, k, s, p, up, h, w in SHAPES:
        conv = _Conv(cin, cout, k, s, p, bias=True, bn_eps=1e-3, up=up, f16=True).init(rng, dev)
        x = (torch.randn((h * w, 2 * cin), device=dev) * 0.5).to(torch.float16)
        conv(x, (1, h, w, cin))  # warm-up
        reps = 5
        rd(None, 0, 1)
        for _ in range(reps):
            conv(x, (1, h, w, cin))
        _lib.check(0 if rd(buf.ctypes.data, max_ctas, 1) == nf else -1, "p3d_dense_trace_read")
        tot = buf.sum(0).astype(np.float64)
        items = tot[0]
        per = {f: tot[i] / items for i, f in enumerate(TRACE_FIELDS) if i > 0}
        row = {"layer": name, "items": int(items / reps), "ctas": int((buf[:, 0] > 0).sum()),
               "cycles_per_item": round(per["cycles"])}
        cons = ("a_full", "b_full", "mma_wait", "epilogue", "stage_free")
        for f in cons:  # mean of the two consumer warpgroups
            row[f] = round((per[f] + per[f + "_1"]) / 2)
        row["other"] = row["cycles_per_item"] - sum(row[f] for f in cons)
        for f in ("prod_a_empty", "prod_b_empty", "epi_warps_wait", "epi_warps_busy"):
            row[f] = round(per[f])
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", action="store_true", help="time every (mode, m_tiles) variant of each layer")
    ap.add_argument("--tf32", action="store_true", help="also time the round-1 tf32-pair kernels")
    ap.add_argument("--trace", action="store_true", help="per-layer wait breakdown of the -DP3D_DENSE_TRACE build")
    args = ap.parse_args()
    if args.trace:
        return trace()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    rng = np.random.default_rng(0)
    H = W = 180
    shapes = SHAPES
    variants = [(0, 0)] + ([(0, 1), (0, 2), (1, 1), (1, 2)] if args.variants else [])
    for name, cin, cout, k, s, p, up, h, w in shapes:
        oh, ow = (h * up, w * up) if up > 1 else ((h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1)
        flops = 2.0 * oh * ow * cin * cout * (1 if up > 1 else k * k)
        conv = _Conv(cin, cout, k, s, p, bias=True, bn_eps=1e-3, up=up, f16=True).init(rng, dev)
        x = (torch.randn((h * w, 2 * cin), device=dev) * 0.5).to(torch.float16)
        for mode, mt in variants:
            if mode == 1 and mt == 0:
                continue
            us = graph_time(lambda: conv(x, (1, h, w, cin), mode=mode, m_tiles=mt))
            print(json.dumps({"layer": name, "kernel": "f16", "mode": mode, "m_tiles": mt, "us": round(us, 1),
                              "gflop": round(flops / 1e9, 2), "algorithmic_tflops": round(flops / us / 1e6, 1)}), flush=True)
        if args.tf32:
            conv32 = _Conv(cin, cout, k, s, p, bias=True, bn_eps=1e-3, up=up, f16=False).init(rng, dev)
            x32 = torch.randn((h * w, 2 * cin), device=dev)
            us = graph_time(lambda: conv32(x32, (1, h, w, cin)))
            print(json.dumps({"layer": name, "kernel": "tf32", "us": round(us, 1), "gflop": round(flops / 1e9, 2),
                              "algorithmic_tflops": round(flops / us / 1e6, 1)}), flush=True)
    net = DenseRPNHead(in_channels=256).init_weight(seed=1, device=dev)
    bev = torch.randn((1, 256, H, W), device=dev)
    print(json.dumps({"whole_head_us": round(graph_time(lambda: net(bev), 3), 1), "kernel": "f16",
                      "env": {k: v for k, v in os.environ.items() if k.startswith("P3D_DENSE")}}), flush=True)
    # pieces of the head
    s, shape = net._trunk(bev)
    bp = net._batched_params(dev)
    mid, _, _ = bp["big"](s, shape)
    pbuf = net._heads_conv_p(s, shape, bp, dev)
    # heads_big_conv_us + final_convs_us: the unfused heads (image written, read back by p3d_head_out_conv_f16);
    # fused_conv_us + tap_sum_us: what forward runs when net.fused_heads(bp)
    print(json.dumps({"trunk_us": round(graph_time(lambda: net._trunk(bev), 3), 1),
                      "heads_big_conv_us": round(graph_time(lambda: bp["big"](s, shape), 3), 1),
                      "final_convs_us": round(graph_time(lambda: net._final_convs(mid, shape, bp["big"].cout, bp, bp["planes"], dev), 3), 1),
                      "fused_conv_us": round(graph_time(lambda: net._heads_conv_p(s, shape, bp, dev), 3), 1),
                      "tap_sum_us": round(graph_time(lambda: net._tap_sum(pbuf, bp, dev), 3), 1),
                      "fused_heads": net.fused_heads(bp),
                      "nchw_to_h16_us": round(graph_time(lambda: dc.nchw_to_pixel_h16(bev), 3), 1)}), flush=True)
    if args.tf32:
        net32 = DenseRPNHead(in_channels=256, f16=False).init_weight(seed=1, device=dev)
        print(json.dumps({"whole_head_us": round(graph_time(lambda: net32(bev), 3), 1), "kernel": "tf32"}), flush=True)


if __name__ == "__main__":
    main()
