"""Camera-to-BEV lifting of BEVDet-style models on the device: LSSViewTransformer
(paddle3d/models/transformers/bevdet_transformer.py, PARITY UNPINNED: restated from BEVDet's class, whose
get_lidar_coor(sensor2ego, ego2global, cam2imgs, post_rots, post_trans, bda) takes a 3x3 bda) from the depth net's
output on, and LSSHotPath, the same forward as one CUDA graph that serves every calibration.

    camera descriptor H2D -> p3d_lss_prepare (frustum geometry fused with the rank keys; sort / scan)
    -> p3d_lss_depth_feat (depth softmax + feature permute) -> p3d_bev_pool_v2_dev ([B, C * Z, Y, X], count on the device)
"""
import numpy as np
import torch

from .frame import GraphFrame
from .ops import bev_pool_v2 as bp


class LSSViewTransformer:
    """grid_config: dict with 'x', 'y', 'z' = [lower, upper, interval] and 'depth' = [start, stop, step]; input_size =
    (H_in, W_in) of the image; the feature maps are input_size // downsample.  out_channels = C of tran_feat.
    accelerate=True (BEVDet's pre_compute): the ranks are kept and recomputed only when the camera matrices change."""

    def __init__(self, grid_config, input_size, downsample, out_channels, accelerate=False, device="cuda"):
        self.device = torch.device(device)
        xyz = [grid_config[k] for k in ("x", "y", "z")]
        self.grid_lower_bound = torch.Tensor([c[0] for c in xyz])
        self.grid_interval = torch.Tensor([c[2] for c in xyz])
        self.grid_size = torch.Tensor([(c[1] - c[0]) / c[2] for c in xyz])
        self.grid = [int(v) for v in self.grid_size]  # X, Y, Z
        self.out_channels = int(out_channels)
        self.accelerate = bool(accelerate)
        self.create_frustum(grid_config["depth"], input_size, downsample)
        self._cache = None  # accelerate: (camera descriptor, prepared ranks)

    def create_frustum(self, depth_cfg, input_size, downsample):
        """The frustum's three axes, built on the host with the reference's expressions and uploaded once."""
        H_in, W_in = input_size
        self.H, self.W = H_in // downsample, W_in // downsample
        d = torch.arange(*depth_cfg, dtype=torch.float)
        x = torch.linspace(0, W_in - 1, self.W, dtype=torch.float)
        y = torch.linspace(0, H_in - 1, self.H, dtype=torch.float)
        self.D = d.numel()
        self.axes_host = (d, x, y)
        self.axes = tuple(a.to(self.device) for a in self.axes_host)

    def grid_args(self):
        return self.grid_lower_bound.tolist(), self.grid_interval.tolist(), self.grid

    def bev_feat_shape(self, B):
        X, Y, Z = self.grid
        return (B, Z, Y, X, self.out_channels)

    def descriptor(self, sensor2ego, cam2imgs, post_rots, post_trans, bda):
        """Device camera descriptor (ops.bev_pool_v2.pack_cameras)."""
        return torch.from_numpy(bp.pack_cameras(sensor2ego, cam2imgs, post_rots, post_trans, bda)).to(self.device)

    def _prepare(self, desc, B, N, with_coor=False):
        return bp.lss_prepare(desc, *self.axes, B, N, *self.grid_args(), with_coor=with_coor)

    def get_lidar_coor(self, sensor2ego, ego2global, cam2imgs, post_rots, post_trans, bda):
        """Ego-frame frustum points [B, N, D, H, W, 3] fp32 on the device (ego2global is unused, as in the reference).
        This is p3d_lss_prepare with its coor output: the rank preparation (sort, scan) runs too and its ranks are
        discarded; callers that pool should call voxel_pooling_v2 / view_transform / forward, which never write coor."""
        B, N = np.shape(sensor2ego)[:2]
        return self._prepare(self.descriptor(sensor2ego, cam2imgs, post_rots, post_trans, bda), B, N, with_coor=True)[6]

    def voxel_pooling_v2(self, coor, depth, feat):
        """coor [B, N, D, H, W, 3], depth [B, N, D, H, W], feat [B, N, C, H, W] -> [B, C * Z, Y, X]; no point inside the grid
        gives zeros, as the reference's dummy tensor."""
        B, N, C, H, W = feat.shape
        prepared = bp.voxel_pooling_prepare_v2(coor, *self.grid_args())
        feat = feat.permute(0, 1, 3, 4, 2).contiguous()
        return bp.bev_pool_v2_dev(depth.contiguous(), feat, prepared, self.bev_feat_shape(B), planar=True)

    def ranks(self, mats, B, N):
        """Prepared ranks of the camera matrices mats = (sensor2ego, cam2imgs, post_rots, post_trans, bda); with accelerate,
        the cached ranks when the descriptor equals the last one."""
        packed = bp.pack_cameras(*mats)
        if self.accelerate and self._cache is not None and np.array_equal(self._cache[0], packed):
            return self._cache[1]
        prepared = self._prepare(torch.from_numpy(packed).to(self.device), B, N)
        if self.accelerate:
            self._cache = (packed, prepared)
        return prepared

    def view_transform(self, input, depth, tran_feat):
        """input = [x [B, N, C_in, H, W], sensor2ego, ego2global, cam2imgs, post_rots, post_trans, bda]; depth [B*N, D, H, W]
        (softmax taken), tran_feat [B*N, C, H, W] -> [B, C * Z, Y, X]."""
        B, N = input[0].shape[:2]
        prepared = self.ranks(_mats(input), B, N)
        feat = tran_feat.view(B * N, self.out_channels, self.H, self.W).permute(0, 2, 3, 1).contiguous()
        return bp.bev_pool_v2_dev(depth.contiguous(), feat, prepared, self.bev_feat_shape(B), planar=True)

    def forward(self, input, logits, tran_feat):
        """From the depth net's output: logits [B*N, D, H, W] and tran_feat [B*N, C, H, W] -> [B, C * Z, Y, X]."""
        B, N = input[0].shape[:2]
        prepared = self.ranks(_mats(input), B, N)
        depth, feat = bp.lss_depth_feat(logits, tran_feat)
        return bp.bev_pool_v2_dev(depth, feat, prepared, self.bev_feat_shape(B), planar=True)


def _mats(input):
    """(sensor2ego, cam2imgs, post_rots, post_trans, bda) of a view_transform input list."""
    return input[1], input[3], input[4], input[5], input[6]


class CameraFrame(GraphFrame):
    """A frame of B samples of N cameras from the depth net's output (logits, tran_feat: device inputs) as captured CUDA
    graphs on its own stream.  The camera descriptor is a device buffer refreshed by an H2D copy at the head of the rank
    stage, so any calibration replays the same graphs.  The frame graph is the rank stage and _frame(); with
    vt.accelerate, a graph "ranks" (replayed only when the camera matrices differ from the last ones) and the graph
    "frame" of the rest.  A subclass defines _frame()."""

    def __init__(self, vt, B, N, device="cuda", stream=None):
        super().__init__(device, stream)
        self.vt, self.B, self.N = vt, B, N
        nd = B * N * bp.CAM_FLOATS + B * 9
        self.h_desc = torch.zeros((nd,), dtype=torch.float32).pin_memory()
        self.desc = torch.zeros((nd,), dtype=torch.float32, device=self.device)
        D, H, W, C = vt.D, vt.H, vt.W, vt.out_channels
        self.logits = torch.zeros((B * N, D, H, W), dtype=torch.float32, device=self.device)
        self.tran_feat = torch.zeros((B * N, C, H, W), dtype=torch.float32, device=self.device)
        self.depth = torch.empty_like(self.logits)
        self.feat = torch.empty((B * N, H, W, C), dtype=torch.float32, device=self.device)
        self.prepared, self.last = None, None
        self.done = torch.cuda.Event()

    # ---- stages, as they are captured
    def _ranks(self):
        self.desc.copy_(self.h_desc, non_blocking=True)
        self.prepared = self.vt._prepare(self.desc, self.B, self.N)

    def _full(self, *args):
        self._ranks()
        return self._frame(*args)

    def _parts(self):
        return {"ranks": self._ranks, "frame": self._frame} if self.vt.accelerate else {"frame": self._full}

    def capture(self, warmup=1, count_nodes=False):
        """Warm up eagerly (sizes the workspaces), then capture the graphs.  count_nodes: node counts by type of the
        graphs in self.graph_nodes."""
        self.last = None
        return super().capture(warmup, count_nodes)

    def launch(self, mats, logits=None, tran_feat=None):
        """Enqueue one frame on self.stream.  mats = (sensor2ego, cam2imgs, post_rots, post_trans, bda) on the host;
        logits / tran_feat: device tensors copied into the frame's inputs (None: already written there)."""
        self._launch(mats, logits, tran_feat, "frame")

    def _launch(self, mats, logits, tran_feat, frame, host_inputs=None):
        """launch() replaying the graph named frame (with accelerate: after the rank graph when the cameras changed);
        host_inputs: called once the previous frame is done, to write further pinned inputs the graph uploads."""
        packed = bp.pack_cameras(*mats)
        self.done.synchronize()  # the previous frame's H2D has read h_desc and its D2H has landed
        if host_inputs is not None:
            host_inputs()
        self.stream.wait_stream(torch.cuda.current_stream(self.device))  # inputs written on the caller's stream
        with torch.cuda.stream(self.stream):
            if logits is not None:
                self.logits.copy_(logits, non_blocking=True)
            if tran_feat is not None:
                self.tran_feat.copy_(tran_feat, non_blocking=True)
            if not self.vt.accelerate:
                self.h_desc.copy_(torch.from_numpy(packed))
            elif self.last is None or not np.array_equal(self.last, packed):
                self.h_desc.copy_(torch.from_numpy(packed))
                self.graphs["ranks"].replay()
                self.last = packed
            self.graphs[frame].replay()
            self.out = self.outs[frame]
            self.done.record(self.stream)


class LSSHotPath(CameraFrame):
    """LSSViewTransformer.forward for B samples of N cameras as one captured CUDA graph (CameraFrame): descriptor H2D,
    ranks, softmax / permute, memset + pool.  launch() enqueues a frame; infer() waits for it and returns the BEV tensor
    with counts = (n_kept, n_intervals), copied back in one D2H inside the rank stage."""

    def __init__(self, vt, B, N, device="cuda", stream=None):
        super().__init__(vt, B, N, device, stream)
        self.h_counts = torch.zeros((2,), dtype=torch.int32).pin_memory()
        X, Y, Z = vt.grid
        self.bev = torch.empty((B, Z * vt.out_channels, Y, X), dtype=torch.float32, device=self.device)

    # ---- stages, as they are captured
    def _ranks(self):
        super()._ranks()
        self.h_counts.copy_(self.prepared[5], non_blocking=True)

    def _frame(self):
        bp.lss_depth_feat(self.logits, self.tran_feat, self.depth, self.feat)
        bp.bev_pool_v2_dev(self.depth, self.feat, self.prepared, self.vt.bev_feat_shape(self.B), planar=True, out=self.bev)

    def infer(self, mats, logits=None, tran_feat=None):
        """One frame, waited for: returns (bev [B, C * Z, Y, X] device tensor owned by the frame, counts (n_kept,
        n_intervals))."""
        self.launch(mats, logits, tran_feat)
        self.done.synchronize()
        return self.bev, tuple(int(v) for v in self.h_counts)
