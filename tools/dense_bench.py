#!/usr/bin/env python
"""Per-layer timing of the dense RPN / neck / CenterHead (SURVEY §8f-1) at the C3 shapes (BEV [1, 256, 180, 180]).

Graph-replayed, one JSON line per distinct layer shape and kernel variant with its algorithmic TFLOP/s (2 * MACs of the
convolution; the kernels execute 3 fp16 MMAs per product), then the whole head.  Needs a GPU:
    python tools/dense_bench.py [--variants] [> dense_layers.jsonl]
"""
import argparse
import json
import os
import sys

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", action="store_true", help="time every (mode, m_tiles) variant of each layer")
    ap.add_argument("--tf32", action="store_true", help="also time the round-1 tf32-pair kernels")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    rng = np.random.default_rng(0)
    H = W = 180
    shapes = [  # (name, cin, cout, k, stride, pad, up, h, w)
        ("backbone0 256->128 s1", 256, 128, 3, 1, 1, 1, H, W), ("backbone0 128->128", 128, 128, 3, 1, 1, 1, H, W),
        ("backbone1 128->256 s2", 128, 256, 3, 2, 1, 1, H, W), ("backbone1 256->256", 256, 256, 3, 1, 1, 1, H // 2, W // 2),
        ("neck 1x1 128->256", 128, 256, 1, 1, 0, 1, H, W), ("neck deconv 256->256 x2", 256, 256, 2, 2, 0, 2, H // 2, W // 2),
        ("shared 512->64", 512, 64, 3, 1, 1, 1, H, W), ("heads 64->2304 (36 batched)", 64, 2304, 3, 1, 1, 1, H, W),
    ]
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
    print(json.dumps({"trunk_us": round(graph_time(lambda: net._trunk(bev), 3), 1),
                      "heads_big_conv_us": round(graph_time(lambda: bp["big"](s, shape), 3), 1),
                      "final_convs_us": round(graph_time(lambda: net._final_convs(mid, shape, bp["big"].cout, bp, bp["planes"], dev), 3), 1),
                      "nchw_to_h16_us": round(graph_time(lambda: dc.nchw_to_pixel_h16(bev), 3), 1)}), flush=True)
    if args.tf32:
        net32 = DenseRPNHead(in_channels=256, f16=False).init_weight(seed=1, device=dev)
        print(json.dumps({"whole_head_us": round(graph_time(lambda: net32(bev), 3), 1), "kernel": "tf32"}), flush=True)


if __name__ == "__main__":
    main()
