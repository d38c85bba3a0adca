"""CenterPoint-pillars inference on one GPU, nuScenes (configs/centerpoint/centerpoint_pillars_02voxel_nuscenes_10sweep.yml,
synth.CP_PILLARS with CONFIG) and KITTI (configs/centerpoint/centerpoint_pillars_016voxel_kitti.yml, synth.CP_PILLARS_KITTI
with CONFIG_KITTI), composed from this repository's kernels (the nuScenes sizes shown):

    hard_voxelize (0.2 m pillars, 20 points) -> PillarFeatureNet with two PFNLayers (one fused launch) -> pillar rows as
    fp16 pairs -> pixel fp16-pair image [512 x 512 x 64] -> SecondBackbone + SecondFPN (a 2x2 stride-2 conv, a 1x1 conv
    and a 2x2 transposed conv into one 128 x 128 x 384 image) + CenterHead (dense_head.DenseRPNHead, 6 tasks, 70 planes)
    -> centerpoint_postprocess_device -> boxes

CenterPointPillarsHotPath captures everything between the H2D copy of the points and the D2H copy of the boxes as one
CUDA graph (frame.CapturedFrame), optionally starting with the device merge of raw sweeps (sweep_input), or for the KITTI
model with the camera frustum cull of a raw scan (sweep_input=frame.KITTI_INPUT: infer_kitti, infer_kitti_many; the
boxes become KITTI labels through kitti.centerpoint_to_lidar_boxes and kitti.to_kitti).

The KITTI model reads 100 points per pillar (pillar_feature_net2 then launches p3d_pillar_feature_net2_wide), has no
velocity head (7-column boxes) and two tasks, [Car] and [Pedestrian, Cyclist]; its head runs at half the 432 x 496 grid.

PARITY UNPINNED: the model values (CONFIG, synth.CP_PILLARS, synth.CENTERPOINT_PILLARS_TEST_CFG) are recalled from
Paddle3D's yml and det3d's nusc_centerpoint_pp_02voxel_two_pfn_10sweep, which it descends from; they were not checked
against either file.  CONFIG_KITTI, synth.CP_PILLARS_KITTI and synth.CP_PILLARS_KITTI_TEST_CFG are recalled from
centerpoint_pillars_016voxel_kitti.yml in the same way."""
import numpy as np
import torch

from . import synth
from .dense_head import COMMON_HEADS, DenseRPNHead, SecondTrunk
from .frame import CapturedFrame, ResultSlot
from .ops import centerpoint_postprocess as cpp
from .ops import pillar_encoder as pe
from .ops import sparse_nn as sp
from .ops import voxelize as vox
from .pointpillars import grid_size

# PARITY UNPINNED (see the module docstring)
CONFIG = dict(
    pfn=dict(feat_channels=(64, 64), bn_eps=1e-3),
    backbone=dict(out_channels=(64, 128, 256), layer_nums=(3, 5, 5), downsample_strides=(2, 2, 2)),
    fpn=dict(out_channels=(128, 128, 128), upsample_strides=(0.5, 1, 2), use_conv_for_no_stride=True),
    head=dict(tasks=tuple(synth.CENTERPOINT_TASKS), share_conv_channel=64),
    test=synth.CENTERPOINT_PILLARS_TEST_CFG,
)
# PARITY UNPINNED (centerpoint_pillars_016voxel_kitti.yml, recalled): PillarFeatureNet(in 4, feat_channels [64, 64],
# with_distance False); SecondBackbone out [64, 128, 256], layer_nums [3, 5, 5], strides [2, 2, 2]; SecondFPN out
# [128, 128, 128], upsample strides [1, 2, 4]; CenterHead share_conv 64, tasks [Car], [Pedestrian, Cyclist], common_heads
# reg 2, height 1, dim 3, rot 2 (no vel)
CONFIG_KITTI = dict(
    pfn=dict(feat_channels=(64, 64), bn_eps=1e-3),
    backbone=dict(out_channels=(64, 128, 256), layer_nums=(3, 5, 5), downsample_strides=(2, 2, 2)),
    fpn=dict(out_channels=(128, 128, 128), upsample_strides=(1, 2, 4), use_conv_for_no_stride=True),
    head=dict(tasks=tuple(synth.CP_PILLARS_KITTI_TASKS), share_conv_channel=64,
              common_heads=(("reg", 2), ("height", 1), ("dim", 3), ("rot", 2))),
    test=synth.CP_PILLARS_KITTI_TEST_CFG,
)


class CenterPointPillars:
    """Seeded CenterPoint-pillars model: PillarFeatureNet(in 5, feat_channels [64, 64]): PFNLayer Linear(F + 5 -> 32) +
    BN + ReLU, concat with the pillar max to 64, PFNLayer Linear(64 -> 64) + BN + ReLU, max (no bias, BatchNorm1D eps
    1e-3); PointPillarsScatter to ny x nx x 64; DenseRPNHead (SecondBackbone [3, 5, 5] / strides [2, 2, 2], SecondFPN
    upsample strides [0.5, 1, 2], CenterHead with 6 tasks) at a quarter of the grid.  model_cfg=CONFIG_KITTI (with
    synth.CP_PILLARS_KITTI) is the KITTI model: PFN in 4, FPN upsample strides [1, 2, 4], two velocity-free tasks, the head
    at half the grid."""

    def __init__(self, cfg=None, model_cfg=None):
        self.cfg = dict(cfg or synth.CP_PILLARS)
        self.mc = model_cfg or CONFIG
        mc = self.mc
        self.grid = grid_size(self.cfg)
        self.F = self.cfg["point_dim"]
        c1, c2 = mc["pfn"]["feat_channels"]
        self.pfn_channels = (c1 // 2, c2)  # a PFNLayer that is not the last one halves its units (pillar_encoder.py)
        self.C = c2
        b, f, h = mc["backbone"], mc["fpn"], mc["head"]
        self.head = DenseRPNHead(in_channels=self.C, out_channels=b["out_channels"], layer_nums=b["layer_nums"],
                                 downsample_strides=b["downsample_strides"], fpn_out_channels=f["out_channels"],
                                 upsample_strides=f["upsample_strides"], tasks=h["tasks"],
                                 share_conv_channel=h["share_conv_channel"], bev_depth=1,
                                 common_heads=h.get("common_heads", COMMON_HEADS))
        self.test_cfg = dict(mc["test"])
        self.label_off = synth.label_offsets(list(h["tasks"]))
        self.feat_hw, self.cat_hw = self._feature_sizes()
        self.pfn = [dict(eps=mc["pfn"]["bn_eps"]) for _ in range(2)]  # parameters: init_weight or load_state_dict
        self.device = None

    def _feature_sizes(self):
        """[(H, W) after each backbone block], (H, W) of the FPN concat (= the head's)."""
        h, w = self.grid[1], self.grid[0]
        sizes = []
        for blk in self.head.blocks:
            for c in blk:
                h, w = (h + 2 * c.padding - c.k) // c.stride + 1, (w + 2 * c.padding - c.k) // c.stride + 1
            sizes.append((h, w))
        cat = {SecondTrunk.deblock_out_hw(de, hh, ww) for (hh, ww), de in zip(sizes, self.head.deblocks)}
        if len(cat) != 1:
            raise ValueError("model config: the FPN deblocks give different sizes %s" % sorted(cat))
        return sizes, cat.pop()

    def init_weight(self, seed=0, device="cuda", bn_gain=1.0):
        """device=None: numpy parameters only (enough for export_numpy / the CPU arm).  bn_gain multiplies every
        BatchNorm gamma (the convention of dense_head.DenseRPNHead.init_weight)."""
        rng = np.random.default_rng(seed)
        eps = self.mc["pfn"]["bn_eps"]
        self.pfn = []
        for fan_in, c in self.pfn_shapes():
            self.pfn.append(dict(weight=synth.kaiming_uniform(rng, (fan_in, c), fan_in),
                                 gamma=np.full(c, bn_gain, np.float32), beta=np.zeros(c, np.float32),
                                 mean=np.zeros(c, np.float32), var=np.ones(c, np.float32), eps=eps))
        self.head.init_weight(seed=seed + 1, device=device, bn_gain=bn_gain)
        return self.derive(device)

    def derive(self, device):
        """The device images of the PFN parameters (self.pfn: per layer Linear weight [in, out] and BatchNorm1D
        statistics): the weights and the folded BN.  Called after new parameters, seeded or loaded; the head derives its
        own (DenseRPNHead.derive)."""
        self.device = None if device is None else torch.device(device)
        if device is not None:
            self.pfn_dev = [dict(l, weight=torch.from_numpy(l["weight"]).to(device)) for l in self.pfn]
            self.pfn_folded = [pe.fold_bn(l["gamma"], l["beta"], l["mean"], l["var"], l["eps"], device) for l in self.pfn]
        return self

    def pfn_shapes(self):
        """Linear weight shapes [in, out] of the two PFN layers."""
        return [(self.F + 5, self.pfn_channels[0]), (2 * self.pfn_channels[0], self.pfn_channels[1])]

    def state_dict(self):
        """Parameters under Paddle3D's names and in its layouts (checkpoint.centerpoint_pillars)."""
        from . import checkpoint
        return checkpoint.state_dict(checkpoint.centerpoint_pillars(self))

    def load_state_dict(self, sd, device=None):
        """Load Paddle3D parameters (checkpoint.load_state_dict: all checked before any is assigned) and re-derive every
        device image on `device` (default: the model's; None keeps numpy parameters only)."""
        from . import checkpoint
        device = self.device if device is None else device
        checkpoint.load_state_dict(checkpoint.centerpoint_pillars(self), sd, device)
        self.head.derive(device)
        self.head.loaded = True
        return self.derive(device)

    def export_numpy(self):
        return dict(self.head.export_numpy(), pfn=self.pfn)

    # ---- per frame, device in / device out
    def encode(self, points):
        """points [n, F] -> (pixel fp16-pair BEV image [ny * nx, 2 C], its shape (1, ny, nx, C), coors [V, 4], num [1])."""
        cfg = self.cfg
        voxels, co, npv, nv = vox.hard_voxelize(points, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"],
                                                cfg["max_voxels"])
        coors = torch.nn.functional.pad(co, (1, 0))  # (batch 0, z, y, x)
        feats = pe.pillar_feature_net2(voxels, npv, coors, self.pfn_dev, cfg["voxel_size"], cfg["point_cloud_range"],
                                       num_voxels=nv, folded=self.pfn_folded)
        nx, ny = self.grid
        image, shape = sp.sparse_coo_tensor(coors, feats, [1, 1, ny, nx, self.C], num=nv).to_pixel_h16()
        return image, shape, coors, nv

    def dense(self, image, shape):
        """Pixel fp16-pair BEV image -> dict name -> per-task [1, k, H / 4, W / 4] fp32 head planes."""
        return self.head.forward_h16(image, shape)

    def postprocess(self, h):
        return cpp.centerpoint_postprocess_heads(h, self.cfg["voxel_size"][:2], self.cfg["point_cloud_range"],
                                                 self.test_cfg, self.label_off)

    def calibrate_heatmap_bias(self, points, target_frac=0.014):
        """DenseRPNHead.calibrate_heatmap_bias on this frame's pixel image: ~1.4 % of the cells above the score
        threshold (SURVEY.md §8d).  Weights stay seeded and are exported unchanged to the CPU arm.  Raises on weights
        loaded from a checkpoint."""
        if self.head.loaded:
            raise RuntimeError("calibrate_heatmap_bias moves the heat-map biases of seeded random weights; this model's "
                               "weights were loaded from a checkpoint and are kept as trained")
        image, shape, _, _ = self.encode(points)
        self.head.calibrate_heatmap_bias(image, self.test_cfg["score_threshold"], target_frac, shape=shape)
        return self

    def head_planes(self):
        return self.head.head_planes()

    def flops(self):
        """Algorithmic flops (2 x MACs) of the dense part at the model's grid: backbone, FPN and head (shared conv, the
        ConvModules (36 nuScenes, 10 KITTI), the output convs)."""
        out = dict(backbone=0.0, fpn=0.0)
        h, w = self.grid[1], self.grid[0]
        for blk in self.head.blocks:
            for c in blk:
                h, w = (h + 2 * c.padding - c.k) // c.stride + 1, (w + 2 * c.padding - c.k) // c.stride + 1
                out["backbone"] += 2.0 * h * w * c.cin * c.cout * c.k * c.k
        for (h, w), de in zip(self.feat_hw, self.head.deblocks):
            oh, ow = SecondTrunk.deblock_out_hw(de, h, w)
            out["fpn"] += 2.0 * oh * ow * de.cin * de.cout * (1 if de.up > 1 else de.k * de.k)
        out.update(self.head.head_flops(*self.cat_hw))
        return out


class CenterPointPillarsHotPath(CapturedFrame):
    """One CenterPoint-pillars frame on one GPU: H2D -> [captured: (sweep merge or camera frustum cull) -> hard_voxelize ->
    PFN -> pixel image -> trunk / head -> centerpoint postprocess] -> D2H of boxes ([6 x 83, 9] nuScenes, [2 x 83, 7]
    KITTI), scores, labels, counts and the status word (fp16-range overflow of the pair path, with sweep input the merge's
    status bits)."""

    def __init__(self, cfg=None, device="cuda:0", seed=0, num_points=None, bn_gain=1.0, model_cfg=None,
                 sweep_input=None, sweep_ring=None, weights=None, share=None):
        """cfg: the point-cloud config (synth.CP_PILLARS by default); sweep_input / sweep_ring: as
        pipeline.CenterPointHotPath (the merged columns are x, y, z, intensity and the time lag: F = 5), or for the KITTI
        model (cfg=synth.CP_PILLARS_KITTI, model_cfg=CONFIG_KITTI) frame.KITTI_INPUT: raw scans culled to the camera
        frustum on the device (infer_kitti, infer_kitti_many).  weights: a
        Paddle3D CenterPoint-pillars checkpoint (a `.pdparams` path or a state dict, see checkpoint.py) instead of the
        seeded weights.  share: another frame whose model this one uses (CenterPointSweep's lanes)."""
        super().__init__(cfg or synth.CP_PILLARS, device, num_points, sweep_input, sweep_ring)
        if share is not None:
            self.share_model(share)
        elif weights is None:
            self.model = CenterPointPillars(self.cfg, model_cfg).init_weight(seed=seed, device=self.device, bn_gain=bn_gain)
        else:
            from .checkpoint import as_state_dict
            self.model = CenterPointPillars(self.cfg, model_cfg).load_state_dict(as_state_dict(weights), self.device)
        m = self.model
        self.slot = ResultSlot(len(m.label_off) * m.test_cfg["nms_post_max_size"], 9 if m.head.with_velocity else 7,
                               len(m.label_off) + 1,
                               1 if self.sweep_input is None else 2)

    def forward_device(self):
        m = self.model
        if self.sweep_input is not None:
            self._merge_sweeps()
        image, shape, coors, nv = m.encode(self.points)
        h = m.dense(image, shape)
        boxes, scores, labels, counts = m.postprocess(h)
        status = torch.stack([sp.status_tensor(self.device)[0]] +
                             ([self._merge_status[0]] if self.sweep_input is not None else []))
        return dict(boxes=boxes, scores=scores, labels=labels, counts=counts, num_voxels=nv, coors=coors, head=h,
                    status=status)

    def _calibrate(self):
        self.model.calibrate_heatmap_bias(self.points)

    def state_dict(self):
        return self.model.state_dict()

    def load_state_dict(self, sd):
        """CenterPointPillars.load_state_dict on the frame's device.  Before capture(): a captured graph reads the images
        it was captured with."""
        if self.graph is not None:
            raise RuntimeError("load_state_dict after capture(): load the weights first, then capture")
        self.model.load_state_dict(sd, self.device)
        return self

    def check_status(self, status_host):
        """Raise when the frame's status word reports dropped rows or an activation outside fp16's range (never a silent
        wrong result)."""
        st = [int(v) for v in status_host]
        if len(st) > 1:
            self._check_merge_status(st[1])
        if st[0]:
            raise RuntimeError("CenterPoint-pillars: an activation left fp16's range (|x| >= 65504) on the fp16-pair path")
