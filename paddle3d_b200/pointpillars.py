"""PointPillars KITTI inference on one GPU: the car model (CONFIG with synth.C2:
configs/pointpillars/pointpillars_xyres16_kitti_car.yml, the SECOND v1.5 `car.xyres_16` values) and the two-class
cyclist / pedestrian model (CONFIG_PED_CYCLIST with synth.C2_PED_CYCLIST:
pointpillars_xyres16_kitti_cyclist_pedestrian.yml, the SECOND v1.5 `ped_cycle/xyres_16` values), composed from this
repository's kernels:

    hard_voxelize -> PillarFeatureNet (one fused launch) -> pillar rows as fp16 pairs -> pixel fp16-pair image
    [496 x 432 car, 248 x 296 cyclist / pedestrian] -> SecondBackbone + SecondFPN (dense_head.SecondTrunk) -> SSD head
    (cls | box | dir as ONE 1x1 conv, fp32 planes) -> anchor_head_postprocess (csrc/anchor_postprocess.cu) -> boxes

PointPillarsHotPath captures everything between the H2D copy of the points and the D2H copy of the boxes as one CUDA graph
(frame.CapturedFrame).  With sweep_input=frame.KITTI_INPUT the graph starts with the camera frustum cull of a raw KITTI
scan (infer_kitti / infer_kitti_many; kitti.py builds the planes and writes the label files).  Anchors are constant per model and built once on the host (create_anchors_3d_stride, SECOND's
box_np_ops), as are the voxel-index corners of each anchor's near box (anchor_voxel_corners) the anchor mask reads."""
import numpy as np
import torch

from . import synth
from .dense_head import SecondTrunk, _Conv
from .ops import anchor_postprocess as ahp
from .ops import pillar_encoder as pe
from .ops import sparse_nn as sp
from .ops import voxelize as vox
from .frame import CapturedFrame, ResultSlot

CONFIG = dict(
    pfn_channels=64, pfn_bn_eps=1e-3,
    backbone=dict(out_channels=(64, 128, 256), layer_nums=(3, 5, 5), downsample_strides=(2, 2, 2)),
    fpn=dict(out_channels=(128, 128, 128), upsample_strides=(1, 2, 4), use_conv_for_no_stride=False),
    anchors_per_loc=2, box_code_size=7, num_dir_bins=2,
    anchor=dict(sizes=(1.6, 3.9, 1.56), strides=(0.32, 0.32, 0.0), offsets=(0.16, -39.52, -1.78), rotations=(0.0, 1.57)),
    test=dict(anchor_area_threshold=1, nms_score_threshold=0.05, nms_iou_threshold=0.5, nms_pre_max_size=1000,
              nms_post_max_size=300, post_center_limit_range=[0.0, -39.68, -5.0, 69.12, 39.68, 5.0]),
)

# SECOND v1.5 ped_cycle/xyres_16 (PARITY UNPINNED, like CONFIG): the first block keeps stride 1, so the head runs at the
# full 248 x 296 grid.  One anchor generator per class, in label order (0 cyclist, 1 pedestrian); per location the
# anchors are (class, rotation), R = 4, and the head has R * (2 + 7 + 2) = 44 channels.
_PED_CYCLIST_ANCHOR = dict(strides=(0.16, 0.16, 0.0), offsets=(0.08, -19.76, -1.465), rotations=(0.0, 1.57))
CONFIG_PED_CYCLIST = dict(
    pfn_channels=64, pfn_bn_eps=1e-3,
    backbone=dict(out_channels=(64, 128, 256), layer_nums=(3, 5, 5), downsample_strides=(1, 2, 2)),
    fpn=dict(out_channels=(128, 128, 128), upsample_strides=(1, 2, 4), use_conv_for_no_stride=False),
    num_classes=2, anchors_per_loc=4, box_code_size=7, num_dir_bins=2,
    anchors=[dict(_PED_CYCLIST_ANCHOR, sizes=(0.6, 1.76, 1.73)),    # cyclist
             dict(_PED_CYCLIST_ANCHOR, sizes=(0.6, 0.8, 1.73))],    # pedestrian
    test=dict(anchor_area_threshold=1, nms_score_threshold=0.05, nms_iou_threshold=0.5, nms_pre_max_size=1000,
              nms_post_max_size=300, post_center_limit_range=[0.0, -19.84, -2.5, 47.36, 19.84, 0.5]),
)


def grid_size(cfg):
    """(nx, ny) of the pillar grid: 432 x 496 for synth.C2."""
    pcr, vs = cfg["point_cloud_range"], cfg["voxel_size"]
    return (int(round((pcr[3] - pcr[0]) / vs[0])), int(round((pcr[4] - pcr[1]) / vs[1])))


def create_anchors_3d_stride(feature_size, sizes, anchor_strides, anchor_offsets, rotations, dtype=np.float32):
    """SECOND box_np_ops.create_anchors_3d_stride: feature_size [D, H, W] -> [D, H, W, n_sizes, n_rot, 7] anchors
    (x, y, z, w, l, h, theta), order (z, y, x, size, rot)."""
    x_stride, y_stride, z_stride = anchor_strides
    x_offset, y_offset, z_offset = anchor_offsets
    z_centers = np.arange(feature_size[0], dtype=dtype) * z_stride + z_offset
    y_centers = np.arange(feature_size[1], dtype=dtype) * y_stride + y_offset
    x_centers = np.arange(feature_size[2], dtype=dtype) * x_stride + x_offset
    sizes = np.reshape(np.array(sizes, dtype=dtype), [-1, 3])
    rotations = np.array(rotations, dtype=dtype)
    rets = list(np.meshgrid(x_centers, y_centers, z_centers, rotations, indexing="ij"))
    tile_shape = [1] * 5
    tile_shape[-2] = int(sizes.shape[0])
    for i in range(len(rets)):
        rets[i] = np.tile(rets[i][..., np.newaxis, :], tile_shape)[..., np.newaxis]
    sizes = np.reshape(sizes, [1, 1, 1, -1, 1, 3])
    tile_size_shape = list(rets[0].shape)
    tile_size_shape[3] = 1
    rets.insert(3, np.tile(sizes, tile_size_shape))
    return np.transpose(np.concatenate(rets, axis=-1), [2, 1, 0, 3, 4, 5])


def anchor_voxel_corners(anchors, voxel_size, point_cloud_range, grid):
    """SECOND's anchor-mask geometry, computed once per model: rbbox2d_to_near_bbox (the axis-aligned box of (w, l), swapped
    when |theta| folded into [0, pi) is nearer pi/2 than 0) and fused_get_anchors_area's floor / clamp to voxel indices.
    anchors [A, 7] -> int32 [A, 4] (x_min, y_min, x_max, y_max)."""
    rb = anchors[:, [0, 1, 3, 4, 6]]
    rots = rb[:, -1]
    folded = np.abs(rots - np.floor(rots / np.pi + 0.5) * np.pi)  # limit_period(rots, 0.5, pi)
    cond = (folded > np.pi / 4)[:, np.newaxis]
    centre_dims = np.where(cond, rb[:, [0, 1, 3, 2]], rb[:, :4])
    near = np.concatenate([centre_dims[:, :2] - centre_dims[:, 2:] / 2, centre_dims[:, :2] + centre_dims[:, 2:] / 2], -1)
    out = np.zeros(near.shape, dtype=np.int32)
    out[:, 0] = np.floor((near[:, 0] - point_cloud_range[0]) / voxel_size[0])
    out[:, 1] = np.floor((near[:, 1] - point_cloud_range[1]) / voxel_size[1])
    out[:, 2] = np.floor((near[:, 2] - point_cloud_range[0]) / voxel_size[0])
    out[:, 3] = np.floor((near[:, 3] - point_cloud_range[1]) / voxel_size[1])
    out[:, [0, 2]] = np.clip(out[:, [0, 2]], 0, grid[0] - 1)
    out[:, [1, 3]] = np.clip(out[:, [1, 3]], 0, grid[1] - 1)
    return out


class PointPillars:
    """Seeded PointPillars model: PillarFeatureNet (one PFNLayer 9 -> 64, no bias, BatchNorm1D eps 1e-3), SecondTrunk and
    the SSD head as one 384 -> R (C + 9) 1x1 conv with bias, C classes and R anchors per location (output channels:
    cls [R x C] | box [R x 7] | dir [R x 2], channel a * K + k of each group belonging to anchor (y * W + x) * R + a;
    car: 384 -> 20)."""

    def __init__(self, cfg=None, model_cfg=None):
        self.cfg = dict(cfg or synth.C2)
        self.mc = model_cfg or CONFIG
        mc = self.mc
        self.grid = grid_size(self.cfg)
        self.F = self.cfg["point_dim"]
        self.C = mc["pfn_channels"]
        self.trunk = SecondTrunk(self.C, mc["backbone"]["out_channels"], mc["backbone"]["layer_nums"],
                                 mc["backbone"]["downsample_strides"], mc["fpn"]["out_channels"],
                                 mc["fpn"]["upsample_strides"], mc["fpn"]["use_conv_for_no_stride"])
        R, self.num_classes = mc["anchors_per_loc"], mc.get("num_classes", 1)
        self.head_channels = R * (self.num_classes + mc["box_code_size"] + mc["num_dir_bins"])
        self.head = _Conv(self.trunk.fpn_channels, self.head_channels, 1, bias=True, relu=False)
        s = mc["backbone"]["downsample_strides"][0]  # the FPN output is at the first block's stride: 248 x 216 (car)
        self.feat_hw = (self.grid[1] // s, self.grid[0] // s)
        # one generator per class, concatenated per location as SECOND's TargetAssigner.generate_anchors does:
        # per location (class, rotation)
        per_class = [create_anchors_3d_stride([1, self.feat_hw[0], self.feat_hw[1]], a["sizes"], a["strides"],
                                              a["offsets"], a["rotations"])
                     for a in (mc["anchors"] if "anchors" in mc else [mc["anchor"]])]
        self.anchors_np = np.concatenate(per_class, axis=3).reshape(-1, 7)
        if len(per_class) != self.num_classes or self.anchors_np.shape[0] != self.feat_hw[0] * self.feat_hw[1] * R:
            raise ValueError("model config: one anchor generator per class, anchors_per_loc anchors per location")
        self.corners_np = anchor_voxel_corners(self.anchors_np, self.cfg["voxel_size"], self.cfg["point_cloud_range"],
                                               self.grid)
        self.pfn = dict(eps=mc["pfn_bn_eps"])  # parameters: init_weight or load_state_dict
        self.device = None
        self.loaded = False  # parameters from a checkpoint (load_state_dict), not seeded

    def init_weight(self, seed=0, device="cuda", bn_gain=1.0):
        """device=None: numpy parameters only (enough for export_numpy / the CPU arm).  bn_gain multiplies every
        BatchNorm gamma (the convention of dense_head.DenseRPNHead.init_weight)."""
        rng = np.random.default_rng(seed)
        C, F = self.C, self.F
        self.pfn = dict(weight=synth.kaiming_uniform(rng, (F + 5, C), F + 5),
                        gamma=np.full(C, bn_gain, np.float32), beta=np.zeros(C, np.float32),
                        mean=np.zeros(C, np.float32), var=np.ones(C, np.float32), eps=self.mc["pfn_bn_eps"])
        for c in self.trunk.convs():
            c.init(rng, device, bn_gain=bn_gain)
        self.head.init(rng, device)
        return self.derive(device)

    def derive(self, device):
        """The device images of the PFN parameters (self.pfn: Linear weight [in, out] and BatchNorm1D statistics), and the
        constant anchors.  Called after new parameters, seeded or loaded; each conv derives its own
        (_Conv.set_parameters)."""
        self.device = None if device is None else torch.device(device)
        if device is not None:
            p = self.pfn
            self.pfn_weight = torch.from_numpy(p["weight"]).to(device)
            self.pfn_folded = pe.fold_bn(p["gamma"], p["beta"], p["mean"], p["var"], p["eps"], device)
            self.anchors = torch.from_numpy(np.ascontiguousarray(self.anchors_np)).to(device)
            self.corners = torch.from_numpy(np.ascontiguousarray(self.corners_np)).to(device)
        return self

    def head_splits(self):
        """(name, output channels) of the SSD head's three convs in the order the one head conv concatenates them."""
        R, mc = self.mc["anchors_per_loc"], self.mc
        return [("cls", R * self.num_classes), ("box", R * mc["box_code_size"]), ("dir", R * mc["num_dir_bins"])]

    def state_dict(self):
        """Parameters under Paddle3D's names and in its layouts (checkpoint.pointpillars)."""
        from . import checkpoint
        return checkpoint.state_dict(checkpoint.pointpillars(self))

    def load_state_dict(self, sd, device=None):
        """Load Paddle3D parameters (checkpoint.load_state_dict: all checked before any is assigned) and re-derive every
        device image on `device` (default: the model's; None keeps numpy parameters only)."""
        from . import checkpoint
        device = self.device if device is None else device
        checkpoint.load_state_dict(checkpoint.pointpillars(self), sd, device)
        self.loaded = True
        return self.derive(device)

    def export_numpy(self):
        return dict(self.trunk.export_numpy(), pfn=self.pfn, head=self.head.np)

    # ---- per frame, device in / device out
    def encode(self, points):
        """points [n, F] -> (pixel fp16-pair BEV image [ny * nx, 2 C], its shape (1, ny, nx, C), coors [V, 4], num [1])."""
        cfg = self.cfg
        voxels, co, npv, nv = vox.hard_voxelize(points, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"],
                                                cfg["max_voxels"])
        coors = torch.nn.functional.pad(co, (1, 0))  # (batch 0, z, y, x)
        p = self.pfn
        feats = pe.pillar_feature_net(voxels, npv, coors, self.pfn_weight, p["gamma"], p["beta"], p["mean"], p["var"],
                                      p["eps"], cfg["voxel_size"], cfg["point_cloud_range"], num_voxels=nv,
                                      folded=self.pfn_folded)
        nx, ny = self.grid
        rows = sp.sparse_coo_tensor(coors, feats, [1, 1, ny, nx, self.C], num=nv)
        image, shape = rows.to_pixel_h16()
        return image, shape, coors, nv

    def dense(self, image, shape):
        """Pixel fp16-pair BEV image -> SSD head planes [1, R (C + 9), H / s, W / s] fp32 (s: the first block's stride)."""
        cat, cshape = self.trunk(image, shape)
        _, planes, _ = self.head(cat, cshape, want_nchw=True)
        return planes

    def postprocess(self, planes, coors, nv, anchor_mask=None, sorted_out=None):
        t = self.mc["test"]
        return ahp.anchor_head_postprocess_device(
            planes, self.anchors, self.corners, coors, nv, self.grid, t["post_center_limit_range"],
            t["anchor_area_threshold"], t["nms_score_threshold"], t["nms_iou_threshold"], t["nms_pre_max_size"],
            t["nms_post_max_size"], anchor_mask=anchor_mask, sorted_out=sorted_out, num_classes=self.num_classes)

    def calibrate_cls_bias(self, points, target_frac=0.02):
        """Seeded weights leave the cls logits near the initial bias, so either almost none or most of the anchors (107,136
        car) would pass the 0.05 score threshold.  This shifts the cls biases of each class so that `target_frac` / C of
        all anchors pass the anchor mask AND the threshold in that class on this frame (at most 2 % together; about 2.1k
        for the car): more than nms_pre_max_size = 1000, so the top-k cut runs, and every class has candidates, so every
        label reaches the output.  Weights stay seeded and are exported unchanged to the CPU arm."""
        if self.loaded:
            raise RuntimeError("calibrate_cls_bias moves the cls biases of seeded random weights; this model's weights "
                               "were loaded from a checkpoint and are kept as trained")
        image, shape, coors, nv = self.encode(points)
        planes = self.dense(image, shape)
        mask = torch.empty((self.anchors.shape[0],), dtype=torch.uint8, device=planes.device)
        self.postprocess(planes, coors, nv, anchor_mask=mask)
        R, C = self.mc["anchors_per_loc"], self.num_classes
        cls = planes[0, :R * C].reshape(R, C, *planes.shape[2:])
        k = int(round(target_frac * self.anchors.shape[0] / C))
        thr = self.mc["test"]["nms_score_threshold"]
        logit_thr = float(np.log(thr / (1.0 - thr)))
        b = self.head.np["bias"].copy()
        for c in range(C):
            logits = cls[:, c].permute(1, 2, 0).reshape(-1)[mask.bool()].float().cpu().numpy()
            if len(logits) > k:
                v = np.sort(logits)[::-1]
                shift = logit_thr - 0.5 * (float(v[k - 1]) + float(v[k]))
            else:
                shift = logit_thr - float(logits.min()) + 1.0 if len(logits) else 0.0
            b[c:R * C:C] = (b[c:R * C:C] + np.float32(shift)).astype(np.float32)  # cls channels a * C + c
        self.head.np["bias"] = b
        self.head.dev["shift"].copy_(torch.from_numpy(b))
        return self

    def flops(self):
        """Algorithmic flops (2 x MACs) of the dense part (backbone, FPN, head) at the model's grid."""
        out = dict(backbone=0.0, fpn=0.0, head=0.0)
        h, w = self.grid[1], self.grid[0]
        sizes = []
        for blk in self.trunk.blocks:
            for c in blk:
                h, w = (h + 2 * c.padding - c.k) // c.stride + 1, (w + 2 * c.padding - c.k) // c.stride + 1
                out["backbone"] += 2.0 * h * w * c.cin * c.cout * c.k * c.k
            sizes.append((h, w))
        for (h, w), de in zip(sizes, self.trunk.deblocks):
            out["fpn"] += 2.0 * (h * de.up) * (w * de.up) * de.cin * de.cout * (1 if de.up > 1 else de.k * de.k)
        out["head"] = 2.0 * self.feat_hw[0] * self.feat_hw[1] * self.head.cin * self.head.cout
        return out


class PointPillarsHotPath(CapturedFrame):
    """One PointPillars frame on one GPU: H2D -> [captured: (camera frustum cull) -> hard_voxelize -> PFN -> pixel image ->
    trunk -> head conv -> anchor postprocess] -> D2H of boxes [300, 7], scores, labels, counts (candidates, rows) and the
    status word (fp16-range overflow of the pair path, with sweep input the cull's status bits)."""

    def __init__(self, cfg=None, device="cuda:0", seed=0, num_points=None, bn_gain=1.0, model_cfg=None, weights=None,
                 share=None, sweep_input=None, sweep_ring=None):
        """cfg: the point-cloud config (synth.C2 by default); model_cfg: the model config (CONFIG by default; synth.C2 with
        CONFIG is the car model, synth.C2_PED_CYCLIST with CONFIG_PED_CYCLIST the cyclist / pedestrian one).  weights: a
        Paddle3D PointPillars checkpoint of that model (a `.pdparams` path or a state dict, see checkpoint.py) instead of
        the seeded weights.  share: another frame whose model this one uses (pipeline.CenterPointSweep's lanes).
        sweep_input / sweep_ring: frame.KITTI_INPUT to run on raw KITTI scans (infer_kitti, infer_kitti_many), culled
        to the camera frustum on the device into the num_points rows the model reads."""
        super().__init__(cfg or synth.C2, device, num_points, sweep_input, sweep_ring)
        if share is not None:
            self.share_model(share)
        elif weights is None:
            self.model = PointPillars(self.cfg, model_cfg).init_weight(seed=seed, device=self.device, bn_gain=bn_gain)
        else:
            from .checkpoint import as_state_dict
            self.model = PointPillars(self.cfg, model_cfg).load_state_dict(as_state_dict(weights), self.device)
        self.slot = ResultSlot(self.model.mc["test"]["nms_post_max_size"], 7, 2, 1 if self.sweep_input is None else 2)

    def forward_device(self):
        m = self.model
        if self.sweep_input is not None:
            self._merge_sweeps()
        image, shape, coors, nv = m.encode(self.points)
        planes = m.dense(image, shape)
        boxes, scores, labels, counts = m.postprocess(planes, coors, nv)
        if self.sweep_input is None:
            status = sp.status_tensor(self.device).clone()
        else:
            status = torch.stack([sp.status_tensor(self.device)[0], self._merge_status[0]])
        return dict(boxes=boxes, scores=scores, labels=labels, counts=counts, num_voxels=nv, coors=coors, planes=planes,
                    status=status)

    def _calibrate(self):
        self.model.calibrate_cls_bias(self.points)

    def state_dict(self):
        return self.model.state_dict()

    def load_state_dict(self, sd):
        """PointPillars.load_state_dict on the frame's device.  Before capture(): a captured graph reads the images it
        was captured with."""
        if self.graph is not None:
            raise RuntimeError("load_state_dict after capture(): load the weights first, then capture")
        self.model.load_state_dict(sd, self.device)
        return self

    def check_status(self, status_host):
        """Raise when the frame's status word reports that an activation left fp16's range, or with sweep input that the
        cull kept more rows than num_points (never a silent wrong result)."""
        if len(status_host) > 1:
            self._check_merge_status(int(status_host[1]))
        if int(status_host[0]):
            raise RuntimeError("PointPillars: an activation left fp16's range (|x| >= 65504) on the fp16-pair path")
