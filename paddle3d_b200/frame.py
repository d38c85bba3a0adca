"""Plumbing of the captured hot-path frames, shared by every model: CUDA-graph capture on a frame's own stream, the pinned
result slot its boxes are read back through, the schedule of frames in flight over several lanes, and CapturedFrame,
the LiDAR frame (points in, boxes out) of pipeline.CenterPointHotPath, pointpillars.PointPillarsHotPath and
centerpoint_pillars.CenterPointPillarsHotPath.  The camera frames build on GraphFrame in lss.py."""
import collections
import ctypes as C

import numpy as np
import torch

from . import raw

_IDENTITY = np.eye(4)

def count_graph_nodes(graph):
    """Node counts by type of a torch.cuda.CUDAGraph captured with keep_graph=True, {"kernel": .., "memcpy": ..,
    "memset": .., "other": ..} (cudaGraphGetNodes / cudaGraphNodeGetType); None when the runtime cannot be queried."""
    try:  # a debugging aid must not take the pipeline down
        rt = raw.cudart()
        g = C.c_void_p(int(graph.raw_cuda_graph()))
        n = C.c_size_t(0)
        if rt.cudaGraphGetNodes(g, None, C.byref(n)) != 0:
            return None
        nodes = (C.c_void_p * n.value)()
        if rt.cudaGraphGetNodes(g, nodes, C.byref(n)) != 0:
            return None
        names = {0: "kernel", 1: "memcpy", 2: "memset"}  # cudaGraphNodeType
        out = {"kernel": 0, "memcpy": 0, "memset": 0, "other": 0}
        for i in range(n.value):
            t = C.c_int(0)
            if rt.cudaGraphNodeGetType(C.c_void_p(nodes[i]), C.byref(t)) != 0:
                return None
            out[names.get(t.value, "other")] += 1
        return out
    except Exception:  # noqa: BLE001
        return None


def copy_rows(dst, src, width):
    """cudaMemcpy2DAsync of the first `width` bytes of every row of src into the rows of dst on the current stream (one
    memcpy node of a captured graph)."""
    rows = src.shape[0]
    if dst.shape[0] != rows or width > dst.stride(0) * dst.element_size() or width > src.stride(0) * src.element_size():
        raise ValueError("copy_rows: %d bytes of %s rows into %s rows" % (width, tuple(src.shape), tuple(dst.shape)))
    rc = raw.cudart().cudaMemcpy2DAsync(dst.data_ptr(), dst.stride(0) * dst.element_size(), src.data_ptr(),
                                        src.stride(0) * src.element_size(), width, rows, 3,  # cudaMemcpyDeviceToDevice
                                        torch.cuda.current_stream(src.device).cuda_stream)
    if rc != 0:
        raise RuntimeError("cudaMemcpy2DAsync failed (cudaError %d)" % rc)


class ResultSlot:
    """Pinned host copy of one frame's result: boxes [rows, box_dims], scores, labels, counts (counts[-1] = the valid
    rows) and the frame's status word."""

    def __init__(self, rows, box_dims, n_counts, n_status):
        self.shape = (rows, box_dims, n_counts, n_status)
        self.boxes = torch.empty((rows, box_dims), dtype=torch.float32).pin_memory()
        self.scores = torch.empty((rows,), dtype=torch.float32).pin_memory()
        self.labels = torch.empty((rows,), dtype=torch.int64).pin_memory()
        self.counts = torch.empty((n_counts,), dtype=torch.int32).pin_memory()
        self.status = torch.zeros((n_status,), dtype=torch.int32).pin_memory()

    def copy_from(self, out):
        """Enqueue the D2H copies of a frame's device outputs (a dict with the five names) on the current stream."""
        self.counts.copy_(out["counts"], non_blocking=True)
        self.status.copy_(out["status"], non_blocking=True)
        self.boxes.copy_(out["boxes"], non_blocking=True)
        self.scores.copy_(out["scores"], non_blocking=True)
        self.labels.copy_(out["labels"], non_blocking=True)

    def read(self, check_status, copied, clone=False):
        """Wait for `copied` (the stream or event after the copies), raise from check_status(self.status), and return
        (boxes [K], scores [K], labels [K]): views of the slot, valid until its next copy, or with clone=True their
        clones."""
        copied.synchronize()
        check_status(self.status)
        k = int(self.counts[-1])
        if clone:
            return self.boxes[:k].clone(), self.scores[:k].clone(), self.labels[:k].clone()
        return self.boxes[:k], self.scores[:k], self.labels[:k]

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in (self.boxes, self.scores, self.labels, self.counts, self.status))


class ResultSlotOwner:
    """Mixin of a frame whose latency-mode result slot is self.slot: h_counts and h_status, the host counts and status
    word of the last frame read back through it."""
    h_counts = property(lambda self: self.slot.counts)
    h_status = property(lambda self: self.slot.status)


class StagedUpload:
    """The double-buffered input upload of a lane whose frames are in flight: the H2D of frame i + 1's inputs runs on a
    copy stream while frame i computes.  Two staging sets shaped like the lane's input buffers `bufs` on the device and,
    with pinned=True, two on the host; `staged[k]` is recorded after the H2D into set k, `consumed[k]` after unstage has
    copied set k into bufs."""

    def __init__(self, bufs, pinned=False):
        self.bufs = list(bufs)
        self.stream = torch.cuda.Stream(self.bufs[0].device)
        self.dev = [[torch.empty_like(b) for b in self.bufs] for _ in range(2)]
        self.host = [[torch.empty(b.shape, dtype=b.dtype, pin_memory=True) for b in self.bufs] for _ in range(2)] \
            if pinned else None
        self.rows = [None, None]  # per set: the leading rows of each buffer its payload fills
        self._staged = [torch.cuda.Event() for _ in range(2)]
        self._consumed = [torch.cuda.Event() for _ in range(2)]

    def stage(self, k, fill, first_use):
        """Enqueue the H2D of one payload into set k on the copy stream: fill(dev, host) enqueues the copies into the
        set's device buffers dev on the current stream (host: the set's pinned buffers, which fill writes first; None
        without them) and returns the leading rows of each buffer it wrote (None: all).  Unless first_use (the set's
        first use since the lane last drained), the copy stream first waits until the set's previous payload is consumed
        and, with pinned staging, the host until that payload's H2D has read the pinned buffers."""
        if not first_use and self.host is not None:
            self._staged[k].synchronize()
        with torch.cuda.stream(self.stream):
            if not first_use:
                self.stream.wait_event(self._consumed[k])
            rows = fill(self.dev[k], None if self.host is None else self.host[k])
            self._staged[k].record(self.stream)
        self.rows[k] = [len(b) for b in self.bufs] if rows is None else rows

    def unstage(self, k, stream):
        """Enqueue on `stream` (the lane's) the wait for set k's H2D and the D2D copies of the rows it holds into bufs."""
        with torch.cuda.stream(stream):
            stream.wait_event(self._staged[k])
            for dst, src, n in zip(self.bufs, self.dev[k], self.rows[k]):
                dst[:n].copy_(src[:n], non_blocking=True)
            self._consumed[k].record(stream)


def in_flight(items, lanes):
    """The schedule of frames in flight over `lanes` lanes: item i runs on lane i % lanes into its result slot
    (i // lanes) & 1; at most lanes + 1 frames are outstanding, and the result of a frame is always read before its
    (lane, slot) is submitted again.  Yields ("submit", i, item, lane, slot) and ("result", i, None, lane, slot) in the
    order they are to be done."""
    pending = collections.deque()
    for i, item in enumerate(items):
        pending.append((i, i % lanes, (i // lanes) & 1))
        yield "submit", i, item, pending[-1][1], pending[-1][2]
        if len(pending) > lanes:
            i0, lane, slot = pending.popleft()
            yield "result", i0, None, lane, slot
    while pending:
        i0, lane, slot = pending.popleft()
        yield "result", i0, None, lane, slot


def run_in_flight(lanes, items, submit):
    """Drive in_flight over the lanes: submit(lane, i, item, slot) enqueues frame i; yields lane._result(slot) per
    frame, in order."""
    for kind, i, item, li, slot in in_flight(items, len(lanes)):
        if kind == "submit":
            submit(lanes[li], i, item, slot)
        else:
            yield lanes[li]._result(slot)


def infer_in_flight(lanes, frames_host):
    """CapturedFrame.infer_many over the lanes: frame i on lane i % len(lanes) (in_flight)."""
    for p in lanes:
        p.prepare_sweep()
    yield from run_in_flight(lanes, frames_host, lambda p, i, pts, k: p._submit(pts, k, i < 2 * len(lanes)))


def kitti_frames(lanes, ring, items):
    """One frame per (cloud [n, 4] fp32 raw scan, planes [6, 4] (kitti.frustum_planes)) over the captured lanes sharing
    `ring` (in_flight), each culled to its camera frustum inside the graph; the H2D of scan j + 1 runs on the ring's copy
    stream while frame j computes.  Yields (boxes, scores, labels) per scan, in order."""
    for p in lanes:
        if p.graph is None or p.ring is not ring or not p.sweep_input["frustum"]:
            raise RuntimeError("infer_kitti_many needs captured lanes with KITTI_INPUT sharing one ring")
        p.prepare_sweep()
    ring.reset()
    yield from run_in_flight(lanes, items, lambda p, i, item, k: p._submit_kitti(item, k))


def stream_frames(lanes, ring, items):
    """One frame per pushed sweep (cloud, global_from_lidar, timestamp) over the captured lanes sharing `ring` (in_flight);
    the H2D of sweep j + 1 runs on the ring's copy stream while frame j computes.  Yields (boxes, scores, labels) per
    sweep, in order."""
    for p in lanes:
        if p.graph is None or p.ring is not ring:
            raise RuntimeError("infer_stream needs captured lanes with sweep input sharing one ring")
        p.prepare_sweep()
    ring.reset()
    yield from run_in_flight(lanes, items, lambda p, i, item, k: p._submit_sweep(ring.push(*item), k))


class GraphFrame:
    """A frame captured as CUDA graphs on its own stream.  A subclass defines _full(), one eager pass of the whole frame,
    and _parts(): graph name -> the stages that graph captures, a callable returning the device outputs it leaves (or
    None).  After capture(): graphs (name -> CUDAGraph), outs (name -> those outputs) and, with count_nodes, graph_nodes
    (the node counts by type summed over the graphs; None when they could not be read)."""

    def __init__(self, device, stream=None):
        self.device = torch.device(device)
        self.stream = stream or torch.cuda.Stream(self.device)
        self.graphs, self.outs, self.graph_nodes, self.out = {}, {}, None, None

    def capture(self, warmup=1, count_nodes=False):
        """Warm up eagerly `warmup` times (sizes the workspaces), then capture each part into its graph."""
        with torch.cuda.stream(self.stream):
            for _ in range(warmup):
                self.out = self._full()
            self.stream.synchronize()
            for name, fn in self._parts().items():
                g = self.graphs[name] = torch.cuda.CUDAGraph(keep_graph=bool(count_nodes))
                with torch.cuda.graph(g, stream=self.stream):
                    self.outs[name] = fn()
        self.stream.synchronize()
        nodes = [count_graph_nodes(g) for g in self.graphs.values()] if count_nodes else [None]
        self.graph_nodes = None if None in nodes else {k: sum(n[k] for n in nodes) for k in nodes[0]}
        return self


# sweep_input of the LiDAR frames: ten nuScenes sweeps of 5 values per point, of which x, y, z, intensity are kept and the
# time lag appended (the 5 columns deploy.preprocess gives the model), close points of earlier sweeps removed within 1 m;
# slot_cap None = 2 x the mean rows per sweep of num_points
SWEEP_INPUT = dict(max_sweeps=10, raw_dim=5, use_dim=4, use_time_lag=True, remove_radius=1.0, slot_cap=None,
                   frustum=False)
# sweep_input of the KITTI PointPillars frames on raw `velodyne/*.bin` scans (infer_kitti / infer_kitti_many): one sweep of
# x, y, z, reflectance, culled on the device to the left colour camera's view frustum (kitti.frustum_planes; Paddle3D's
# RemoveCameraInvisiblePointsKITTI) into the frame's points.  A raw HDL-64E scan holds ~120k points; slot_cap is the
# largest raw scan a frame takes.
KITTI_INPUT = dict(max_sweeps=1, raw_dim=4, use_dim=4, use_time_lag=False, remove_radius=1.0, slot_cap=196608,
                   frustum=True)


class CapturedFrame(ResultSlotOwner, GraphFrame):
    """A LiDAR frame captured as one graph, "frame" (self.graph): forward_device() of the points in self.points, with the
    public infer() / infer_many() calls and their pinned result slots, and the sweep input (infer_sweeps /
    infer_stream).  A subclass calls __init__, sets self.model (or its own model fields and share_model /
    calibrate_head) and self.slot = ResultSlot(...) (n_status counting the merge's status word with sweep input), and
    defines forward_device() (returning at least boxes / scores / labels / counts / status, counts[-1] the number of
    valid rows; with sweep input it starts with _merge_sweeps()) and check_status()."""

    def __init__(self, cfg, device, num_points=None, sweep_input=None, sweep_ring=None):
        """sweep_input: None (the frame reads merged clouds from self.points) or a dict over SWEEP_INPUT's keys: the frame
        then starts with the device merge (ops.sweep_merge) of raw sweeps held in a SweepRing into self.points (num_points
        rows, NaN beyond the merged ones); see infer_sweeps / infer_stream.  sweep_ring: a ring shared with other lanes
        (pipeline.CenterPointSweep); default: an own ring of max_sweeps + 1 slots."""
        super().__init__(device)
        self.cfg = dict(cfg)
        self.n = int(num_points or self.cfg["num_points"])
        self.F = self.cfg["point_dim"]
        self.points = torch.zeros((self.n, self.F), dtype=torch.float32, device=self.device)  # static input
        self.graph = self._upload = None
        self.sweep_input = self.ring = None
        if sweep_input is not None:
            self._init_sweep_input(dict(SWEEP_INPUT, **sweep_input), sweep_ring)

    def share_model(self, other):
        self.model = other.model

    def calibrate_head(self, points_dev):
        """The model's head calibration on this frame (_calibrate).  Call before capture()."""
        with torch.cuda.stream(self.stream):
            self.points.copy_(points_dev)
            self._calibrate()
        self.stream.synchronize()
        return self

    def _full(self):
        return self.forward_device()

    def _parts(self):
        return {"frame": self.forward_device}

    def capture(self, warmup=2, count_nodes=False):
        """Warm up (sizes the workspaces) on the side stream, then capture the frame into self.graph.  count_nodes: keep
        the cudaGraph_t and store its node counts in self.graph_nodes (count_graph_nodes)."""
        super().capture(warmup, count_nodes)
        self.graph, self.out = self.graphs["frame"], self.outs["frame"]
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
            self.slot.copy_from(self.out)
        return self.slot.read(self.check_status, self.stream)

    # ---- public end-to-end call for a sweep of frames: same per-frame work, copies overlapped with compute
    def prepare_sweep(self):
        """Staged upload of the points, pinned result slots and events of infer_many (allocated once; pinned allocations
        cost milliseconds, so callers that time a sweep call this first)."""
        if self._upload is not None:
            return self
        self._upload = StagedUpload([self.points])
        self._slots = [ResultSlot(*self.slot.shape) for _ in range(2)]
        self._done = [torch.cuda.Event() for _ in range(2)]  # results of slot k are on the host
        return self

    def _submit(self, pts, k, first_use):
        """Enqueue one frame of a sweep into slot k: H2D into staging set k on the copy stream, its D2D into the points,
        graph replay, D2H of the results."""
        def fill(dev, host):
            dev[0].copy_(pts, non_blocking=True)
        self._upload.stage(k, fill, first_use)
        self._upload.unstage(k, self.stream)
        with torch.cuda.stream(self.stream):
            self.graph.replay()
            self._slots[k].copy_from(self.out)
            self._done[k].record(self.stream)

    def _result(self, k):
        return self._slots[k].read(self.check_status, self._done[k], clone=True)

    def infer_many(self, frames_host):
        """frames_host: iterable of pinned [n, F] fp32 tensors.  Yields (boxes, scores, labels) per frame, in order.

        Every frame still pays its own H2D copy and its own D2H read-back; the H2D of frame i+1 runs on a copy
        stream while frame i computes (two device staging buffers, two pinned result slots), and the host reads the
        results of frame i after it has submitted frame i+1.  pipeline.CenterPointSweep runs several such lanes side by
        side."""
        if self.graph is None:
            raise RuntimeError("infer_many needs a captured pipeline: call capture() first")
        yield from infer_in_flight([self], frames_host)

    # ---- sweep input (sweep_input=...): raw sweeps in a SweepRing, merged on the device inside the captured frame
    def _init_sweep_input(self, si, ring):
        from . import sweep_ring
        from .ops import sweep_merge as sm
        si["use_dim"] = sm.columns(si["use_dim"], si["raw_dim"])
        if len(si["use_dim"]) + bool(si["use_time_lag"]) != self.F:
            raise ValueError("sweep_input gives %d columns per point, the model reads %d"
                             % (len(si["use_dim"]) + bool(si["use_time_lag"]), self.F))
        K = int(si["max_sweeps"])
        if si["frustum"] and (K != 1 or si["use_time_lag"]):
            raise ValueError("the camera frustum cull takes one sweep without a time lag")
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
        if si["frustum"]:  # the six frustum planes the captured cull reads, staged like the descriptor
            self._planes = torch.zeros((6, 4), dtype=torch.float64, device=self.device)
            self._planes_host = [torch.zeros((6, 4), dtype=torch.float64).pin_memory() for _ in range(3)]

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
        return stream_frames([self], self.ring, items)

    def _submit_sweep(self, j, k):
        """Enqueue the frame keyed by ring sweep j into result slot k: descriptor H2D, graph replay, D2H of the results."""
        read, pushed = self.ring.describe(j, self._desc_view(k))
        st = self.stream
        with torch.cuda.stream(st):
            st.wait_event(pushed)
            self._sweep_desc.copy_(self._desc_host[k], non_blocking=True)
            self.graph.replay()
            self._slots[k].copy_from(self.out)
            self._done[k].record(st)
        self.ring.mark_read(read, self._done[k])

    def _kitti_input(self, cloud, planes):
        """Checked (cloud, planes) of a KITTI frame: nothing is enqueued for a refused one."""
        from . import kitti
        if self.sweep_input is None or not self.sweep_input["frustum"]:
            raise RuntimeError("KITTI frames need a pipeline built with sweep_input=frame.KITTI_INPUT")
        cloud = np.ascontiguousarray(cloud, np.float32)
        if cloud.ndim != 2 or cloud.shape[1] != self.ring.raw_dim or len(cloud) > self.ring.slot_cap:
            raise ValueError("a raw scan must be [n <= %d, %d], got %s" % (self.ring.slot_cap, self.ring.raw_dim,
                                                                           cloud.shape))
        return cloud, kitti.check_planes(planes)

    def infer_kitti(self, cloud, planes):
        """One frame from a raw KITTI scan, latency mode: cloud [n, 4] fp32 (a `velodyne/*.bin`), planes [6, 4] float64
        (kitti.frustum_planes of its calib and image shape).  The rows outside the camera frustum are dropped on the
        device; returns what infer() returns for the culled cloud (LiDAR-frame boxes; kitti.to_kitti makes labels)."""
        cloud, planes = self._kitti_input(cloud, planes)
        from .ops import sweep_merge as sm
        desc = self._desc_view(2)
        self.stream.synchronize()  # the previous frame no longer reads the staging
        desc[:] = np.zeros(1, sm.DESC_DTYPE)
        self._planes_host[2].numpy()[:] = planes
        self.ring.reset()
        self.ring.load(0, cloud, self.stream)
        sm.set_entry(desc[0], 0, len(cloud))

        def upload():
            self._sweep_desc.copy_(self._desc_host[2], non_blocking=True)
            self._planes.copy_(self._planes_host[2], non_blocking=True)
        out = self._infer(upload)
        ev = torch.cuda.Event()
        ev.record(self.stream)
        self.ring.mark_read([0], ev)
        return out

    def infer_kitti_many(self, items):
        """items: iterable of (cloud, planes) as infer_kitti takes them.  Yields (boxes, scores, labels) per scan, in
        order; the H2D of the next scan overlaps the current frame (as infer_many)."""
        if self.graph is None:
            raise RuntimeError("infer_kitti_many needs a captured pipeline: call capture() first")
        return kitti_frames([self], self.ring, items)

    def _submit_kitti(self, item, k):
        """Enqueue the frame of one raw scan into result slot k: scan H2D into the ring, descriptor and plane H2D, graph
        replay, D2H of the results."""
        cloud, planes = self._kitti_input(*item)
        j = self.ring.push(cloud, _IDENTITY, 0.0)
        self._planes_host[k].numpy()[:] = planes  # slot k's previous frame was read back: its H2D is done
        read, pushed = self.ring.describe(j, self._desc_view(k))
        st = self.stream
        with torch.cuda.stream(st):
            st.wait_event(pushed)
            self._sweep_desc.copy_(self._desc_host[k], non_blocking=True)
            self._planes.copy_(self._planes_host[k], non_blocking=True)
            self.graph.replay()
            self._slots[k].copy_from(self.out)
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
        if si["frustum"]:
            sm.merge_frustum_into(self.ring.buf, self._sweep_desc, self._planes, si["use_dim"], self.points,
                                  self._n_merged, self._merge_status)
            return
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
        return self.n * self.F * 4, self.slot.nbytes()
