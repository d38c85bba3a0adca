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
import numpy as np
import torch

from . import synth
from .layers import SparseResNet3D
from .ops import centerpoint_postprocess as cpp
from .ops import sparse_nn as sp
from .ops import voxelize as vox


def _count_graph_nodes(raw_graph):
    """Node counts of a cudaGraph_t by type, through libcudart (ctypes)."""
    import ctypes as C
    rt = C.CDLL("libcudart.so")
    n = C.c_size_t(0)
    g = C.c_void_p(int(raw_graph))
    if rt.cudaGraphGetNodes(g, None, C.byref(n)) != 0:
        return None
    nodes = (C.c_void_p * n.value)()
    if rt.cudaGraphGetNodes(g, nodes, C.byref(n)) != 0:
        return None
    names = {0: "kernel", 1: "memcpy", 2: "memset"}  # cudaGraphNodeType
    out = {"kernel": 0, "memcpy": 0, "memset": 0, "other": 0}
    for i in range(n.value):
        t = C.c_int(0)
        rt.cudaGraphNodeGetType(C.c_void_p(nodes[i]), C.byref(t))
        out[names.get(t.value, "other")] += 1
    return out


class CapturedFrame:
    """Plumbing shared by the captured hot-path frames (CenterPointHotPath, pointpillars.PointPillarsHotPath,
    centerpoint_pillars.CenterPointPillarsHotPath): warm-up and CUDA-graph capture of forward_device() on a side stream,
    the public infer() / infer_many() calls and their pinned result slots, and the sweep input (infer_sweeps /
    infer_stream).  A subclass sets self.device / self.points / self.stream / self.graph = self.out = None (and
    self.sweep_input = self.ring = None, or calls _init_sweep_input and starts forward_device() with _merge_sweeps()),
    calls _alloc_host_outputs, and defines forward_device() (returning at least boxes / scores / labels / counts / status,
    with counts[-1] the number of valid rows) and check_status()."""

    def _alloc_host_outputs(self, rows, box_dims, n_counts, n_status):
        self.h_boxes = torch.empty((rows, box_dims), dtype=torch.float32).pin_memory()
        self.h_scores = torch.empty((rows,), dtype=torch.float32).pin_memory()
        self.h_labels = torch.empty((rows,), dtype=torch.int64).pin_memory()
        self.h_counts = torch.empty((n_counts,), dtype=torch.int32).pin_memory()
        self.h_status = torch.zeros((n_status,), dtype=torch.int32).pin_memory()

    def capture(self, warmup=2, count_nodes=False):
        """Warm up (sizes the workspaces) on the side stream, then capture the frame into a CUDA graph.  count_nodes:
        keep the cudaGraph_t and store its node counts (cudaGraphGetNodes / cudaGraphNodeGetType) in self.graph_nodes =
        {"kernel": .., "memset": .., "memcpy": .., "other": ..}."""
        with torch.cuda.stream(self.stream):
            for _ in range(warmup):
                self.out = self.forward_device()
            self.stream.synchronize()
            self.graph = torch.cuda.CUDAGraph(keep_graph=True) if count_nodes else torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self.stream):
                self.out = self.forward_device()
            self.graph_nodes = None
            if count_nodes:
                try:
                    self.graph_nodes = _count_graph_nodes(self.graph.raw_cuda_graph())
                except Exception:  # noqa: BLE001  (a debugging aid must not take the pipeline down)
                    self.graph_nodes = None
        self.stream.synchronize()
        return self

    def launch(self):
        """Replay the captured frame on the pipeline stream (inputs already in self.points)."""
        with torch.cuda.stream(self.stream):
            self.graph.replay()

    # ---- public end-to-end call: host points in, host boxes out
    def infer(self, points_host):
        """points_host: pinned [n, F] fp32 tensor.  Returns (boxes [K, 9 or 7], scores [K], labels [K]) on the host."""
        return self._infer(lambda: self.points.copy_(points_host, non_blocking=True))

    def _infer(self, upload):
        """One frame in latency mode: upload() enqueues the H2D copies of the inputs on the pipeline stream."""
        with torch.cuda.stream(self.stream):
            upload()
            if self.graph is not None:
                self.graph.replay()
            else:
                self.out = self.forward_device()
            o = self.out
            self.h_counts.copy_(o["counts"], non_blocking=True)
            self.h_status.copy_(o["status"], non_blocking=True)
            self.h_boxes.copy_(o["boxes"], non_blocking=True)
            self.h_scores.copy_(o["scores"], non_blocking=True)
            self.h_labels.copy_(o["labels"], non_blocking=True)
        self.stream.synchronize()
        self.check_status(self.h_status)
        k = int(self.h_counts[-1])
        return self.h_boxes[:k], self.h_scores[:k], self.h_labels[:k]

    # ---- public end-to-end call for a sweep of frames: same per-frame work, copies overlapped with compute
    def prepare_sweep(self):
        """Copy stream, staging buffers, pinned result slots and events of infer_many (allocated once; pinned allocations
        cost milliseconds, so callers that time a sweep call this first)."""
        if getattr(self, "_copy_stream", None) is not None:
            return self
        self._copy_stream = torch.cuda.Stream(self.device)
        self._staging = [torch.empty_like(self.points) for _ in range(2)]
        self._slots = [dict(boxes=torch.empty_like(self.h_boxes).pin_memory(),
                            scores=torch.empty_like(self.h_scores).pin_memory(),
                            labels=torch.empty_like(self.h_labels).pin_memory(),
                            counts=torch.empty_like(self.h_counts).pin_memory(),
                            status=torch.zeros_like(self.h_status).pin_memory()) for _ in range(2)]
        self._staged = [torch.cuda.Event() for _ in range(2)]    # H2D into staging[k] done
        self._consumed = [torch.cuda.Event() for _ in range(2)]  # staging[k] copied into the graph's input
        self._done = [torch.cuda.Event() for _ in range(2)]      # results of slot k are on the host
        return self

    def _submit(self, pts, k, first_use):
        """Enqueue one frame of a sweep into slot k: H2D on the copy stream, graph replay, D2H of the results."""
        cs, st = self._copy_stream, self.stream
        with torch.cuda.stream(cs):
            if not first_use:
                cs.wait_event(self._consumed[k])
            self._staging[k].copy_(pts, non_blocking=True)
            self._staged[k].record(cs)
        with torch.cuda.stream(st):
            st.wait_event(self._staged[k])
            self.points.copy_(self._staging[k], non_blocking=True)
            self._consumed[k].record(st)
            self.graph.replay()
            o, sl = self.out, self._slots[k]
            sl["counts"].copy_(o["counts"], non_blocking=True)
            sl["status"].copy_(o["status"], non_blocking=True)
            sl["boxes"].copy_(o["boxes"], non_blocking=True)
            sl["scores"].copy_(o["scores"], non_blocking=True)
            sl["labels"].copy_(o["labels"], non_blocking=True)
            self._done[k].record(st)

    def _result(self, k):
        self._done[k].synchronize()
        sl = self._slots[k]
        self.check_status(sl["status"])
        n = int(sl["counts"][-1])
        return sl["boxes"][:n].clone(), sl["scores"][:n].clone(), sl["labels"][:n].clone()

    def infer_many(self, frames_host):
        """frames_host: iterable of pinned [n, F] fp32 tensors.  Yields (boxes, scores, labels) per frame, in order.

        Every frame still pays its own H2D copy and its own D2H read-back; the H2D of frame i+1 runs on a copy
        stream while frame i computes (two device staging buffers, two pinned result slots), and the host reads the
        results of frame i after it has submitted frame i+1.  CenterPointSweep runs several such lanes side by side."""
        if self.graph is None:
            raise RuntimeError("infer_many needs a captured pipeline: call capture() first")
        self.prepare_sweep()
        i = -1
        for i, pts in enumerate(frames_host):
            self._submit(pts, i & 1, i < 2)
            if i >= 1:
                yield self._result((i - 1) & 1)
        if i >= 0:
            yield self._result(i & 1)

    # ---- sweep input (sweep_input=...): raw sweeps in a SweepRing, merged on the device inside the captured frame
    def _init_sweep_input(self, si, ring):
        from . import sweep_ring
        from .ops import sweep_merge as sm
        si["use_dim"] = sm.columns(si["use_dim"], si["raw_dim"])
        if len(si["use_dim"]) + bool(si["use_time_lag"]) != self.F:
            raise ValueError("sweep_input gives %d columns per point, the model reads %d"
                             % (len(si["use_dim"]) + bool(si["use_time_lag"]), self.F))
        K = int(si["max_sweeps"])
        if si["slot_cap"] is None:
            si["slot_cap"] = -(-2 * self.n // K // 4) * 4
        if ring is None:
            ring = sweep_ring.SweepRing(K, si["raw_dim"], si["slot_cap"], K + 1, self.device)
        if (ring.max_sweeps, ring.raw_dim, ring.slot_cap) != (K, si["raw_dim"], si["slot_cap"]):
            raise ValueError("the sweep ring does not match sweep_input")
        self.sweep_input, self.ring = si, ring
        nb = K * sm.DESC_DTYPE.itemsize
        self._sweep_desc = torch.zeros((nb,), dtype=torch.uint8, device=self.device)  # read by the captured merge
        self._desc_host = [torch.zeros((nb,), dtype=torch.uint8).pin_memory() for _ in range(3)]
        self._n_merged = torch.zeros((1,), dtype=torch.int32, device=self.device)
        self._merge_status = torch.zeros((1,), dtype=torch.int32, device=self.device)

    def _desc_view(self, k):
        from .ops import sweep_merge as sm
        return self._desc_host[k].numpy().view(sm.DESC_DTYPE)

    def infer_sweeps(self, key, sweeps=()):
        """One frame from raw arrays, latency mode: key [n, raw_dim] fp32, sweeps [(cloud, ref_from_curr | None,
        time_lag)] in merge order, at most max_sweeps - 1 (io.merge_sweeps' arguments).  Returns what infer() returns
        for the merged cloud.  Starts a new stream of the ring."""
        si, ring = self.sweep_input, self.ring
        if si is None:
            raise RuntimeError("infer_sweeps needs a pipeline built with sweep_input")
        if len(sweeps) + 1 > si["max_sweeps"]:
            raise ValueError("%d sweeps exceed max_sweeps = %d" % (len(sweeps) + 1, si["max_sweeps"]))
        from .ops import sweep_merge as sm
        desc = self._desc_view(2)
        self.stream.synchronize()  # the previous frame no longer reads the descriptor staging
        desc[:] = np.zeros(1, sm.DESC_DTYPE)
        ring.reset()
        for e, (cloud, m, lag) in enumerate([(key, None, 0.0)] + list(sweeps)):
            ring.load(e, cloud, self.stream)
            sm.set_entry(desc[e], e, len(cloud), m, lag)

        def upload():
            self._sweep_desc.copy_(self._desc_host[2], non_blocking=True)
        out = self._infer(upload)
        ev = torch.cuda.Event()
        ev.record(self.stream)
        ring.mark_read(range(len(sweeps) + 1), ev)
        return out

    def infer_stream(self, items):
        """items: iterable of (cloud [n, raw_dim] fp32, global_from_lidar 4x4, timestamp [s]), one per sensor sweep.
        Yields one (boxes, scores, labels) per pushed sweep, in order: the frame keyed by that sweep with the
        max_sweeps - 1 previous ones of the stream.  The H2D of the next sweep overlaps the current frame (as infer_many)."""
        if self.graph is None:
            raise RuntimeError("infer_stream needs a captured pipeline: call capture() first")
        return _stream_frames([self], self.ring, items)

    def _submit_sweep(self, j, k):
        """Enqueue the frame keyed by ring sweep j into result slot k: descriptor H2D, graph replay, D2H of the results."""
        read, pushed = self.ring.describe(j, self._desc_view(k))
        st = self.stream
        with torch.cuda.stream(st):
            st.wait_event(pushed)
            self._sweep_desc.copy_(self._desc_host[k], non_blocking=True)
            self.graph.replay()
            o, sl = self.out, self._slots[k]
            for name in ("counts", "status", "boxes", "scores", "labels"):
                sl[name].copy_(o[name], non_blocking=True)
            self._done[k].record(st)
        self.ring.mark_read(read, self._done[k])

    def merged_rows(self):
        """Rows of the last merged cloud (device scalar read back; sweep input only)."""
        self.stream.synchronize()
        return int(self._n_merged.item())

    def _merge_sweeps(self):
        """Enqueue the device merge (ops.sweep_merge) of the frame's sweeps in the ring into self.points."""
        from .ops import sweep_merge as sm
        si = self.sweep_input
        sm.merge_into(self.ring.buf, self._sweep_desc, si["max_sweeps"], si["use_dim"], si["use_time_lag"],
                      si["remove_radius"], self.points, self._n_merged, self._merge_status)

    def _check_merge_status(self, v):
        """Raise when the merge's status bits report a bad descriptor entry or dropped rows."""
        if v:
            from .ops import sweep_merge as sm
            if v & sm.BAD_ENTRY:
                raise RuntimeError("sweep merge: a frame descriptor entry named a slot or row count outside the ring")
            raise RuntimeError("sweep merge: the merged sweeps exceed the point capacity (num_points = %d); rows were "
                               "dropped" % self.n)

    def bytes_per_frame(self):
        h2d = self.n * self.F * 4
        d2h = (self.h_boxes.numel() * 4 + self.h_scores.numel() * 4 + self.h_labels.numel() * 8 + self.h_counts.numel() * 4 +
               self.h_status.numel() * 4)
        return h2d, d2h


def _stream_frames(lanes, ring, items):
    """One frame per pushed sweep (cloud, global_from_lidar, timestamp) over the captured lanes sharing `ring`: frame j
    runs on lane j % len(lanes), result slot (j // len(lanes)) & 1 (CenterPointSweep.plan); the H2D of sweep j + 1 runs
    on the ring's copy stream while frame j computes.  Yields (boxes, scores, labels) per sweep, in order."""
    import collections
    L = len(lanes)
    for p in lanes:
        if p.graph is None or p.ring is not ring:
            raise RuntimeError("infer_stream needs captured lanes with sweep input sharing one ring")
        p.prepare_sweep()
    ring.reset()
    pending = collections.deque()
    for i, (cloud, pose, t) in enumerate(items):
        li, k = CenterPointSweep._lane_slot(i, L)
        lane = lanes[li]
        lane._submit_sweep(ring.push(cloud, pose, t), k)
        pending.append((lane, k))
        if len(pending) > L:
            pl, pk = pending.popleft()
            yield pl._result(pk)
    while pending:
        pl, pk = pending.popleft()
        yield pl._result(pk)


# sweep_input of CenterPointHotPath: ten nuScenes sweeps of 5 values per point, of which x, y, z, intensity are kept
# and the time lag appended (the 5 columns deploy.preprocess gives the model), close points of earlier sweeps removed
# within 1 m; slot_cap None = 2 x the mean rows per sweep of num_points
SWEEP_INPUT = dict(max_sweeps=10, raw_dim=5, use_dim=4, use_time_lag=True, remove_radius=1.0, slot_cap=None)


class CenterPointHotPath(CapturedFrame):
    def __init__(self, cfg=None, device="cuda:0", precision=sp.FP32, seed=0, num_points=None, level_caps=None,
                 head_seed=0, with_head=False, keep_bev=True, bn_gain=1.0, sweep_input=None, sweep_ring=None):
        """sweep_input: None (the frame reads merged clouds from self.points) or a dict over SWEEP_INPUT's keys: the
        frame then starts with the device merge (ops.sweep_merge) of raw sweeps held in a SweepRing into self.points
        (num_points rows, NaN beyond the merged ones); see infer_sweeps / infer_stream.  sweep_ring: a ring shared
        with other lanes (CenterPointSweep); default: an own ring of max_sweeps + 1 slots."""
        self.cfg = dict(cfg or synth.C3)
        self.device = torch.device(device)
        self.n = int(num_points or self.cfg["num_points"])
        self.F = self.cfg["point_dim"]
        self.test_cfg = dict(synth.CENTERPOINT_TEST_CFG)
        self.label_off = synth.label_offsets()
        self.net = SparseResNet3D(self.F, self.cfg["voxel_size"], self.cfg["point_cloud_range"])
        self.net.init_weight(seed=seed, device=self.device, bn_gain=bn_gain).set_precision(precision)
        V = self.cfg["max_voxels"]
        self.net.set_level_caps(level_caps or [3 * V, 3 * V, 2 * V, V])
        h = synth.centerpoint_head_outputs(head_seed)
        self.head_host = h
        self.head = {k: [torch.from_numpy(x).to(self.device) for x in v] for k, v in h.items()}
        # with_head: run the dense RPN / neck / CenterHead (dense_head.DenseRPNHead, SURVEY §8f-1) on the BEV tensor and
        # feed ITS outputs to the postprocess instead of the resident synthetic head tensors (parity-green per layer and
        # as a small network; this whole-frame composition has not been timed yet, hence off by default)
        self.dense = None
        if with_head:
            from .dense_head import DenseRPNHead
            self.dense = DenseRPNHead(in_channels=128 * 2).init_weight(seed=seed + 1, device=self.device, bn_gain=bn_gain)
        # keep_bev=False (with the fp16-pair dense head): the sparse rows go straight into the pixel fp16-pair image the RPN
        # reads; the reference's fp32 NCHW BEV tensor is then not materialised in the frame (bev_nchw() rebuilds it on demand)
        self.keep_bev = keep_bev or self.dense is None or not self.dense.f16
        self.points = torch.zeros((self.n, self.F), dtype=torch.float32, device=self.device)  # static input
        self.graph = None
        self.out = None
        self.stream = torch.cuda.Stream(self.device)
        self.sweep_input = self.ring = None
        if sweep_input is not None:
            self._init_sweep_input(dict(SWEEP_INPUT, **sweep_input), sweep_ring)
        self._alloc_host_outputs(len(self.label_off) * self.test_cfg["nms_post_max_size"], 9, len(self.label_off) + 1,
                                 5 if self.sweep_input is None else 6)

    # ---- one frame, enqueued on the current stream, device in / device out
    def forward_device(self):
        cfg, tc = self.cfg, self.test_cfg
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
        boxes, scores, labels, counts = cpp.centerpoint_postprocess_device(
            h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], cfg["voxel_size"][:2],
            cfg["point_cloud_range"], tc["post_center_limit_range"], self.label_off, tc["down_ratio"],
            tc["score_threshold"], tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"], True)
        return dict(bev=bev, bev_h16=bev_h16, boxes=boxes, scores=scores, labels=labels, counts=counts, num_voxels=nv,
                    coors=coors, mean=mean, status=status)

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
        DenseRPNHead.calibrate_heatmap_bias).  Call before capture()."""
        if self.dense is None:
            return self
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
        """frame_cls: the hot-path class of each lane (default CenterPointHotPath; pointpillars.PointPillarsHotPath)."""
        if lanes < 1:
            raise ValueError("lanes >= 1")
        frame_cls = frame_cls or CenterPointHotPath
        first = frame_cls(**kw)
        if kw.get("sweep_input") is not None and kw.get("sweep_ring") is None:
            # one ring for all lanes, K + lanes slots: a slot is reused only after its last reader's result was read
            from .sweep_ring import SweepRing
            si = first.sweep_input
            first.ring = SweepRing(si["max_sweeps"], si["raw_dim"], si["slot_cap"], si["max_sweeps"] + lanes, first.device)
            kw = dict(kw, sweep_ring=first.ring)
        self.lanes = [first]
        for _ in range(lanes - 1):
            p = frame_cls(**kw)
            p.share_model(first)  # one model: calibration / weight loading happens once, on lane 0
            self.lanes.append(p)
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
    def _lane_slot(i, lanes):
        return i % lanes, (i // lanes) & 1

    @staticmethod
    def plan(n_frames, lanes):
        """The order of operations of infer_many for a sweep of n_frames: ("submit", frame, lane, slot) / ("result", frame,
        lane, slot) tuples.  Frame i runs on lane i % lanes, slot (i // lanes) & 1; at most lanes + 1 frames are
        outstanding, and the result of a frame is always read before its (lane, slot) is submitted again
        (tests/test_sweep_plan.py checks these invariants without a GPU)."""
        import collections
        pending = collections.deque()
        for i in range(n_frames):
            pending.append((i,) + CenterPointSweep._lane_slot(i, lanes))
            yield ("submit",) + pending[-1]
            if len(pending) > lanes:
                yield ("result",) + pending.popleft()
        while pending:
            yield ("result",) + pending.popleft()

    def infer_stream(self, items):
        """As CenterPointHotPath.infer_stream (one result per pushed sweep, in order), with the lanes sharing one sweep
        ring and len(self) frames computing concurrently."""
        return _stream_frames(self.lanes, self.lanes[0].ring, items)

    def infer_many(self, frames_host):
        """As CenterPointHotPath.infer_many (pinned host frames in, host results out, in order), with len(self) frames
        computing concurrently: frame i runs on lane i % lanes, slot (i // lanes) & 1 (see plan())."""
        import collections
        L = len(self.lanes)
        for p in self.lanes:
            if p.graph is None:
                raise RuntimeError("infer_many needs captured lanes: call capture() first")
            p.prepare_sweep()
        pending = collections.deque()
        for i, pts in enumerate(frames_host):
            li, k = self._lane_slot(i, L)
            lane = self.lanes[li]
            lane._submit(pts, k, i < 2 * L)
            pending.append((lane, k))
            if len(pending) > L:
                pl, pk = pending.popleft()
                yield pl._result(pk)
        while pending:
            pl, pk = pending.popleft()
            yield pl._result(pk)
