"""CenterPoint-voxel hot-path frame on one GPU: the public API a user calls (bench.py `e2e`).

    voxelize (+ VoxelMean fused)  ->  SparseResNet3D (21 sparse convs)  ->  dense BEV [1,256,180,180]
    -> dense 2-D RPN + neck + CenterHead (with_head=True; otherwise resident synthetic head tensors)
    -> centerpoint_postprocess -> boxes

Everything between the H2D copy of the points and the D2H copy of the boxes is captured once in a
CUDA graph (data-dependent row counts live in device scalars, buffers are sized by capacity), so a
frame is: cudaMemcpyAsync H2D, one graph launch, cudaMemcpyAsync D2H.
Call sites mirrored: CenterPoint.extract_feat (centerpoint.py:126-138) and
CenterHead.predict_by_custom_op (center_head.py:294-339).
"""
import torch

from . import synth
from .frame import (SWEEP_INPUT, CapturedFrame, ResultSlot, infer_in_flight, in_flight, kitti_frames,  # noqa: F401
                    stream_frames)
from .layers import SparseResNet3D
from .ops import centerpoint_postprocess as cpp
from .ops import sparse_nn as sp
from .ops import voxelize as vox


class CenterPointHotPath(CapturedFrame):
    def __init__(self, cfg=None, device="cuda:0", precision=sp.FP32, seed=0, num_points=None, level_caps=None,
                 head_seed=0, with_head=False, keep_bev=True, bn_gain=1.0, sweep_input=None, sweep_ring=None, weights=None,
                 share=None):
        """sweep_input / sweep_ring: see frame.CapturedFrame.  weights: a Paddle3D CenterPoint-voxel checkpoint (a
        `.pdparams` path or a state dict, see checkpoint.py) instead of the seeded weights; needs with_head=True.
        share: another CenterPointHotPath whose model (weights, packed images) this frame uses, built by it (weights,
        seed, bn_gain and precision are then ignored; CenterPointSweep's lanes)."""
        super().__init__(cfg or synth.C3, device, num_points, sweep_input, sweep_ring)
        if weights is not None and not with_head:
            raise ValueError("weights: a CenterPoint checkpoint holds the dense RPN / neck / CenterHead as well; build the "
                             "frame with with_head=True")
        self.test_cfg = dict(synth.CENTERPOINT_TEST_CFG)
        self.label_off = synth.label_offsets()
        h = synth.centerpoint_head_outputs(head_seed)
        self.head_host = h
        self.head = {k: [torch.from_numpy(x).to(self.device) for x in v] for k, v in h.items()}
        # with_head: run the dense RPN / neck / CenterHead (dense_head.DenseRPNHead, SURVEY §8f-1) on the BEV tensor and
        # feed ITS outputs to the postprocess instead of the resident synthetic head tensors (parity-green per layer and
        # as a small network; this whole-frame composition has not been timed yet, hence off by default)
        if share is not None:
            self.share_model(share)
        else:
            self.net = SparseResNet3D(self.F, self.cfg["voxel_size"], self.cfg["point_cloud_range"])
            self.dense = None
            if with_head:
                from .dense_head import DenseRPNHead
                self.dense = DenseRPNHead(in_channels=128 * 2)
            if weights is None:
                self.net.init_weight(seed=seed, device=self.device, bn_gain=bn_gain)
                if self.dense is not None:
                    self.dense.init_weight(seed=seed + 1, device=self.device, bn_gain=bn_gain)
            else:
                from .checkpoint import as_state_dict
                self.load_state_dict(as_state_dict(weights))
            self.net.set_precision(precision)
            V = self.cfg["max_voxels"]
            self.net.set_level_caps(level_caps or [3 * V, 3 * V, 2 * V, V])
        # keep_bev=False (with the fp16-pair dense head): the sparse rows go straight into the pixel fp16-pair image the RPN
        # reads; the reference's fp32 NCHW BEV tensor is then not materialised in the frame (bev_nchw() rebuilds it on demand)
        self.keep_bev = keep_bev or self.dense is None or not self.dense.f16
        self.slot = ResultSlot(len(self.label_off) * self.test_cfg["nms_post_max_size"], 9, len(self.label_off) + 1,
                               5 if self.sweep_input is None else 6)

    # ---- one frame, enqueued on the current stream, device in / device out
    def forward_device(self):
        cfg = self.cfg
        si = self.sweep_input
        if si is not None:
            self._merge_sweeps()
        mean, coors, npv, nv = vox.voxelize_mean(self.points, cfg["voxel_size"], cfg["point_cloud_range"],
                                                 cfg["max_points"], cfg["max_voxels"], 0)
        bev, bev_h16 = None, None
        if self.keep_bev:
            bev = self.net(mean, coors, 1, num=nv)
            h = self.dense(bev) if self.dense is not None else self.head
        else:
            bev_h16 = self.net(mean, coors, 1, num=nv, pixel_h16=True)
            h = self.dense.forward_h16(*bev_h16)
        # frame status word (ADVICE r1): [fp16-range overflow of the pair-row kernels, overflow flag of each strided level,
        # with sweep input: the merge's status bits]
        status = torch.stack([sp.status_tensor(self.device)[0]] + [c[1] for c in self.net.level_counters] +
                             ([self._merge_status[0]] if si is not None else []))
        boxes, scores, labels, counts = cpp.centerpoint_postprocess_heads(h, cfg["voxel_size"][:2], cfg["point_cloud_range"],
                                                                          self.test_cfg, self.label_off)
        return dict(bev=bev, bev_h16=bev_h16, boxes=boxes, scores=scores, labels=labels, counts=counts, num_voxels=nv,
                    coors=coors, mean=mean, status=status, head=h)

    def bev_nchw(self):
        """The dense BEV tensor [1, 256, H, W] fp32 of the last frame (rebuilt from the pixel fp16-pair image when the
        frame did not materialise it)."""
        if self.out["bev"] is not None:
            self.stream.synchronize()
            return self.out["bev"]
        from .ops import dense_conv as dc
        rows, shape = self.out["bev_h16"]
        with torch.cuda.stream(self.stream):
            out = dc.pixel_h16_to_nchw(rows, shape)
            # pixel rows hold (z, c)-ordered channels (to_pixel_h16); the reference tensor is (c, z)-ordered
            b, h, w, cd = shape
            D = self.dense.bev_depth
            out = out.view(b, D, cd // D, h, w).transpose(1, 2).reshape(b, cd, h, w).contiguous()
        self.stream.synchronize()  # callers read it from other streams
        return out

    def calibrate_head(self, points_dev):
        """Shift the heat-map biases of the (randomly initialised) dense head so that ~1.4 % of the BEV cells of this frame
        score above the threshold, as SURVEY.md §8d specifies for the synthetic workload (see
        DenseRPNHead.calibrate_heatmap_bias).  Call before capture(); raises on weights loaded from a checkpoint."""
        if self.dense is None:
            return self
        if self.dense.loaded:
            raise RuntimeError("calibrate_head moves the heat-map biases of seeded random weights; this frame's weights "
                               "were loaded from a checkpoint and are kept as trained")
        cfg = self.cfg
        with torch.cuda.stream(self.stream):
            self.points.copy_(points_dev)
            mean, coors, npv, nv = vox.voxelize_mean(self.points, cfg["voxel_size"], cfg["point_cloud_range"],
                                                     cfg["max_points"], cfg["max_voxels"], 0)
            bev = self.net(mean, coors, 1, num=nv)
            self.dense.calibrate_heatmap_bias(bev, self.test_cfg["score_threshold"])
        self.stream.synchronize()
        return self

    def check_status(self, status_host):
        """Raise when the frame's device status word reports dropped work (never a silent wrong result)."""
        st = [int(v) for v in status_host]
        n_levels = len(self.net.level_counters)
        if len(st) > 1 + n_levels:
            self._check_merge_status(st[1 + n_levels])
        if st[0]:
            raise RuntimeError("sparse backbone: an activation left fp16's range (|x| >= 65504) on the fp16-pair path; "
                               "run this model with precision TF32X3_SPLIT")
        for lvl, v in enumerate(st[1:1 + n_levels]):
            if v:
                raise RuntimeError("sparse backbone: strided level %d overflowed its row capacity (set_level_caps); "
                                   "output sites were dropped" % (lvl + 1))

    def share_model(self, other):
        self.net, self.dense = other.net, other.dense

    def state_dict(self):
        """The model's parameters under Paddle3D's names and in its layouts (checkpoint.centerpoint_voxel)."""
        from . import checkpoint
        if self.dense is None:
            raise ValueError("state_dict: a frame without the dense head (with_head=False) is not a whole CenterPoint")
        return checkpoint.state_dict(checkpoint.centerpoint_voxel(self.net, self.dense))

    def load_state_dict(self, sd):
        """Load Paddle3D CenterPoint-voxel parameters (checkpoint.load_state_dict: all checked before any is assigned)
        and re-derive every device image.  Before capture(): a captured graph reads the images it was captured with."""
        from . import checkpoint
        if self.dense is None:
            raise ValueError("load_state_dict: a frame without the dense head (with_head=False) is not a whole CenterPoint")
        if self.graph is not None:
            raise RuntimeError("load_state_dict after capture(): load the weights first, then capture")
        checkpoint.load_state_dict(checkpoint.centerpoint_voxel(self.net, self.dense), sd, self.device)
        self.dense.derive(self.device)
        self.dense.loaded = True
        return self

    def export_weights_numpy(self):
        """Weights as plain numpy dicts for the CPU arm (oracle.cpu_reference.CpuFrame)."""
        def conv(l):
            return dict(weight=l.weight.cpu().numpy(), bias=None if l.bias is None else l.bias.cpu().numpy(),
                        stride=l.stride, padding=l.padding)

        def bn(l):
            return dict(gamma=l.weight.cpu().numpy(), beta=l.bias.cpu().numpy(), mean=l._mean.cpu().numpy(),
                        var=l._variance.cpu().numpy(), eps=l.epsilon)

        def block(b):
            return dict(conv1=conv(b.conv1), bn1=bn(b.bn1), conv2=conv(b.conv2), bn2=bn(b.bn2))

        n = self.net
        return dict(conv_input=dict(conv=conv(n.conv_input[0]), bn=bn(n.conv_input[1])),
                    blocks0=[block(b) for b in n.blocks0],
                    stages=[dict(down=dict(conv=conv(d[0]), bn=bn(d[1])), blocks=[block(b) for b in bl]) for d, bl in n.stages],
                    extra=dict(conv=conv(n.extra_conv[0]), bn=bn(n.extra_conv[1])))


class CenterPointSweep:
    """Several frames of a sweep in flight on ONE GPU.

    `lanes` CenterPointHotPath instances share the model (weights, packed images) but own their buffers, workspaces,
    CUDA graph and stream; frames are dealt round-robin.  A frame is a chain of ~70 kernels of very different shapes -
    persistent tensor-core kernels that fill the GPU, and latency-bound ones (voxel hashing, rulebooks, post-processing,
    the tails of every layer) that leave most SMs idle: with a second frame in flight those gaps are filled by the other
    frame's kernels (tools/two_in_flight.py compares one and two lanes).  The latency of one frame does not improve (use CenterPointHotPath.infer for that); results are those of the single-lane pipeline.
    """

    def __init__(self, lanes=2, frame_cls=None, **kw):
        """frame_cls: the hot-path class of each lane (default CenterPointHotPath; pointpillars.PointPillarsHotPath,
        centerpoint_pillars.CenterPointPillarsHotPath).  kw: the frame's arguments; weights= (a checkpoint) is loaded
        once, into lane 0's model, which every lane shares."""
        if lanes < 1:
            raise ValueError("lanes >= 1")
        frame_cls = frame_cls or CenterPointHotPath
        first = frame_cls(**kw)  # weights= (a checkpoint path) is read here, once
        kw.pop("weights", None)
        if kw.get("sweep_input") is not None and kw.get("sweep_ring") is None:
            # one ring for all lanes, K + lanes slots: a slot is reused only after its last reader's result was read
            from .sweep_ring import SweepRing
            si = first.sweep_input
            first.ring = SweepRing(si["max_sweeps"], si["raw_dim"], si["slot_cap"], si["max_sweeps"] + lanes, first.device)
            kw = dict(kw, sweep_ring=first.ring)
        self.lanes = [first]
        for _ in range(lanes - 1):
            # one model: built, loaded and calibrated once, on lane 0; the other lanes build none
            self.lanes.append(frame_cls(share=first, **kw))
        self.device = first.device

    def __len__(self):
        return len(self.lanes)

    def calibrate_head(self, points_dev):
        self.lanes[0].calibrate_head(points_dev)
        return self

    def capture(self, points_dev, **kw):
        for p in self.lanes:
            p.points.copy_(points_dev)
            p.capture(**kw)
        return self

    def prepare_sweep(self):
        for p in self.lanes:
            p.prepare_sweep()
        return self

    def launch(self, i, points_dev):
        """Frame i of a device-resident sweep: copy into lane i % lanes and replay its graph (asynchronous)."""
        p = self.lanes[i % len(self.lanes)]
        with torch.cuda.stream(p.stream):
            p.points.copy_(points_dev, non_blocking=True)
            p.graph.replay()
        return p

    def synchronize(self):
        for p in self.lanes:
            p.stream.synchronize()

    @staticmethod
    def plan(n_frames, lanes):
        """The order of operations of infer_many for a sweep of n_frames: ("submit", frame, lane, slot) / ("result", frame,
        lane, slot) tuples (frame.in_flight: frame i runs on lane i % lanes, slot (i // lanes) & 1; at most lanes + 1
        frames are outstanding, and the result of a frame is always read before its (lane, slot) is submitted again)."""
        for kind, i, _, lane, slot in in_flight(range(n_frames), lanes):
            yield kind, i, lane, slot

    def infer_stream(self, items):
        """As CenterPointHotPath.infer_stream (one result per pushed sweep, in order), with the lanes sharing one sweep
        ring and len(self) frames computing concurrently."""
        return stream_frames(self.lanes, self.lanes[0].ring, items)

    def infer_kitti_many(self, items):
        """As PointPillarsHotPath.infer_kitti_many ((raw scan, frustum planes) items in, host results out, in order), with
        the lanes (built with sweep_input=frame.KITTI_INPUT) sharing one ring and len(self) frames computing
        concurrently."""
        return kitti_frames(self.lanes, self.lanes[0].ring, items)

    def infer_many(self, frames_host):
        """As CenterPointHotPath.infer_many (pinned host frames in, host results out, in order), with len(self) frames
        computing concurrently: frame i runs on lane i % lanes, slot (i // lanes) & 1 (see plan())."""
        if any(p.graph is None for p in self.lanes):
            raise RuntimeError("infer_many needs captured lanes: call capture() first")
        yield from infer_in_flight(self.lanes, frames_host)
