"""BEVFusion (bevf_pp, configs/bevfusion/bevf_pp_2x8_1x_nusc.yaml) from the depth net's output and a LiDAR cloud to boxes:
the seeded model (BEVFusion) and the captured frame (BEVFusionHotPath).

PARITY UNPINNED: every value below is recalled from ADLab's BEVFusion (BEVF_FasterRCNN, cam_stream_lss.py) and mmdet3d
v0.17 (HardVFE, SECOND, SECONDFPN, Anchor3DHead, box3d_multiclass_nms), which bevf_pp descends from; none was checked
against either.  A checkout corrects them here, in one place.  The device entry points this model needs are
ops.pillar_encoder.hard_vfe (the LiDAR encoder), ops.se_gate.se_gate_h16 (the SE_Block after the fusion conv) and
ops.anchor3d_postprocess (the head's decode).

Two deliberate differences from the reference, both PARITY UNPINNED: a camera BEV cell sums its points in sorted order
(bev_pool_v2's rule) where cam_stream_lss sums them with the fp32 cumsum-and-difference trick (equal in exact
arithmetic), and the camera BEV is laid out y rows by x columns like the pillar image (LSS's voxel_pooling writes
[Z, X, Y]; a checkout showing the reference keeps that order changes only the rank key's axis order)."""
import numpy as np
import torch

from .dense_head import SecondTrunk, _Conv
from .frame import ResultSlot, ResultSlotOwner
from .lss import CameraFrame, LSSViewTransformer
from .ops import anchor3d_postprocess as a3d
from .ops import bev_pool_v2 as bp
from .ops import pillar_encoder as pe
from .ops import sparse_nn as sp
from .ops import voxelize as vox
from .ops.se_gate import se_gate_h16

CLASSES = ("car", "truck", "trailer", "bus", "construction_vehicle", "bicycle", "motorcycle", "pedestrian",
           "traffic_cone", "barrier")

CONFIG = dict(
    # LiDAR stream (synth.C4_LIDAR): HardVoxelizer -> HardVFE -> PointPillarsScatter -> SECOND -> SECONDFPN
    voxel_size=(0.25, 0.25, 8.0),
    point_cloud_range=(-50.0, -50.0, -5.0, 50.0, 50.0, 3.0),
    max_points=64,
    max_voxels=40000,
    vfe=dict(in_channels=4, feat_channels=(64, 64), bn_eps=1e-3),
    # camera stream (cam_stream_lss.py): depth bins [4, 45, 1], 900 x 1600 images at downsample 8, camC 64
    dbound=(4.0, 45.0, 1.0),
    image_size=(900, 1600),
    downsample=8,
    cam_channels=64,
    xbound=(-50.0, 50.0, 0.5),
    ybound=(-50.0, 50.0, 0.5),
    zbound=(-5.0, 3.0, 0.5),
    cam_encoder=(1024, 1024, 512, 256),
    cam_bn_eps=1e-5,
    n_cams=6,
    backbone=dict(out_channels=(64, 128, 256), layer_nums=(3, 5, 5), downsample_strides=(2, 2, 2)),
    fpn=dict(out_channels=(128, 128, 128), upsample_strides=(1, 2, 4)),
    # fusion: concat(camera 256, LiDAR 384) -> reduc_conv 3x3 640 -> 384 (BN eps 1e-3, ReLU) -> SE_Block(384)
    fusion_channels=384,
    fusion_bn_eps=1e-3,
    # Anchor3DHead: AlignedAnchor3DRangeGenerator(align_corner=False), sizes (w, l, h), one z per (range, size) pair
    anchor_xy=49.6,
    anchors=(
        ((1.95017717, 4.60718145, 1.72270761), -1.80032795),   # car
        ((2.4560939, 6.73778078, 2.73004906), -1.74440365),    # truck
        ((2.87427237, 12.01320693, 3.81509561), -1.68526504),  # trailer
        ((0.60058911, 1.68452161, 1.27192197), -1.67339111),   # bicycle
        ((0.66344886, 0.7256437, 1.75748069), -1.61785072),    # pedestrian
        ((0.39694519, 0.40359262, 1.06232151), -1.80984986),   # traffic_cone
        ((2.49008838, 0.48578221, 0.98297065), -1.763965),     # barrier
    ),
    rotations=(0.0, 1.57),
    custom_values=(0.0, 0.0),
    feat_size=(200, 200),
    test=dict(nms_pre=1000, score_thr=0.05, nms_thr=0.2, max_num=500, dir_offset=0.7854, dir_limit_offset=0.0),
)


def anchors_per_loc(cfg=CONFIG):
    return len(cfg["anchors"]) * len(cfg["rotations"])


def make_anchors(cfg=CONFIG, feat_size=None):
    """AlignedAnchor3DRangeGenerator(align_corner=False) on an H x W map: [H * W * S * R, 9] fp32 (x, y, z, w, l, h, r,
    then the custom values), anchor ((y * W + x) * S + s) * R + r for size s and rotation r.  The centres are
    linspace(-xy, xy, n + 1)[:n] + half a step, computed in fp64 and rounded once (torch.linspace's fp32 rounding is not
    reproduced)."""
    H, W = feat_size or cfg["feat_size"]
    xy = float(cfg["anchor_xy"])
    xs = np.linspace(-xy, xy, W + 1)
    ys = np.linspace(-xy, xy, H + 1)
    xs = xs[:W] + (xs[1] - xs[0]) / 2
    ys = ys[:H] + (ys[1] - ys[0]) / 2
    S, rots = len(cfg["anchors"]), np.asarray(cfg["rotations"], np.float64)
    R = len(rots)
    out = np.zeros((H, W, S, R, 7 + len(cfg["custom_values"])), np.float64)
    out[..., 0] = xs[None, :, None, None]
    out[..., 1] = ys[:, None, None, None]
    for s, (size, z) in enumerate(cfg["anchors"]):
        out[:, :, s, :, 2] = z
        out[:, :, s, :, 3:6] = size
    out[..., 6] = rots
    out[..., 7:] = 0.0  # mmdet3d leaves the custom columns zero (its `custom[:] = self.custom_values` is commented out)
    return out.reshape(-1, out.shape[-1]).astype(np.float32)


def small_config():
    """The model at test size: a 32 x 32 pillar grid (1 m pillars over +-16 m) and a 16 x 16 x 16 camera grid (2 m cells)
    from 256 x 448 images at downsample 16, so both BEVs are 16 x 16; every channel width and rule as CONFIG."""
    return dict(CONFIG, voxel_size=(1.0, 1.0, 8.0), point_cloud_range=(-16.0, -16.0, -5.0, 16.0, 16.0, 3.0),
                max_voxels=1024, image_size=(256, 448), downsample=16, xbound=(-16.0, 16.0, 2.0),
                ybound=(-16.0, 16.0, 2.0), anchor_xy=15.5, feat_size=(16, 16))


class BEVFusion:
    """Seeded BEVFusion (bevf_pp) at batch 1.  LiDAR: hard_voxelize -> HardVFE -> pixel scatter -> SecondTrunk into
    channels [cam_C, cam_C + 384) of the 640-channel fusion image.  Camera: LSSViewTransformer (depth softmax, pool
    into Z * camC = 1024 channels) -> three 3x3 ConvModules into channels [0, cam_C).  Then reduc_conv (3x3, 640 -> 384,
    BN eps 1e-3, ReLU), SE_Block(384), the Anchor3DHead convs as one 384 -> 294 1x1 conv and anchor3d_postprocess."""

    def __init__(self, cfg=None, accelerate=False, device="cuda"):
        self.cfg = c = dict(cfg or CONFIG)
        self.device = torch.device(device)
        self.N = c["n_cams"]
        pcr, vs = c["point_cloud_range"], c["voxel_size"]
        self.grid = (int(round((pcr[3] - pcr[0]) / vs[0])), int(round((pcr[4] - pcr[1]) / vs[1])))  # (nx, ny)
        grid_cfg = dict(x=list(c["xbound"]), y=list(c["ybound"]), z=list(c["zbound"]), depth=list(c["dbound"]))
        self.vt = LSSViewTransformer(grid_cfg, c["image_size"], c["downsample"], c["cam_channels"], accelerate=accelerate,
                                     device=self.device)
        X, Y, Z = self.vt.grid
        self.pool_C = Z * c["cam_channels"]
        if self.pool_C % 32 or self.pool_C != c["cam_encoder"][0]:
            raise ValueError("the camera encoder takes %d channels, the pool gives %d" % (c["cam_encoder"][0], self.pool_C))
        ce = c["cam_encoder"]
        self.cam_convs = [_Conv(ci, co, 3, 1, 1, bn_eps=c["cam_bn_eps"]) for ci, co in zip(ce[:-1], ce[1:])]
        b, f = c["backbone"], c["fpn"]
        self.F = c["vfe"]["in_channels"]
        self.vfe_C = c["vfe"]["feat_channels"]
        self.trunk = SecondTrunk(self.vfe_C[1], b["out_channels"], b["layer_nums"], b["downsample_strides"],
                                 f["out_channels"], f["upsample_strides"])
        s0 = b["downsample_strides"][0]
        lidar_hw = (self.grid[1] // s0, self.grid[0] // s0)
        if lidar_hw != (Y, X) or tuple(c["feat_size"]) != (Y, X):
            raise ValueError("the LiDAR BEV is %s, the camera BEV %s and feat_size %s: the fusion needs one size (the "
                             "reference's F.interpolate for different sizes is not supported)"
                             % (lidar_hw, (Y, X), tuple(c["feat_size"])))
        self.cam_C = ce[-1]
        self.fuse_C = self.cam_C + self.trunk.fpn_channels
        fc = c["fusion_channels"]
        self.reduc = _Conv(self.fuse_C, fc, 3, 1, 1, bn_eps=c["fusion_bn_eps"])
        self.num_classes, self.R = len(CLASSES), anchors_per_loc(c)
        self.head = _Conv(fc, self.R * (self.num_classes + 9 + 2), 1, bias=True, relu=False)
        self.bev_hw = (Y, X)
        self.anchors_np = make_anchors(c)

    def convs(self):
        return self.cam_convs + self.trunk.convs() + [self.reduc, self.head]

    def init_weight(self, seed=0, device=None):
        """Seeded weights; device=False: numpy parameters only (export_numpy / the CPU arm).  The BN gains keep the seeded
        activations inside fp16's range."""
        rng = np.random.default_rng(seed)
        dev = None if device is False else (device or self.device)
        F, (mid, out) = self.F, self.vfe_C
        eps = self.cfg["vfe"]["bn_eps"]

        def vfe_layer(cin, cout):
            bound = 1.0 / np.sqrt(cin)
            return dict(weight=rng.uniform(-bound, bound, (cin, cout)).astype(np.float32),
                        gamma=np.full(cout, 2.0, np.float32), beta=np.zeros(cout, np.float32),
                        mean=np.zeros(cout, np.float32), var=np.ones(cout, np.float32), eps=eps)
        self.vfe = [vfe_layer(F + 6, mid), vfe_layer(2 * mid, out)]
        for cv in self.cam_convs + self.trunk.convs() + [self.reduc]:
            cv.init(rng, dev, bn_gain=6.0 ** 0.5)
        self.head.init(rng, dev)
        fc = self.cfg["fusion_channels"]
        bound = 1.0 / np.sqrt(fc)
        self.se = dict(weight=rng.uniform(-bound, bound, (fc, fc)).astype(np.float32),
                       bias=rng.uniform(-bound, bound, fc).astype(np.float32))
        if dev is not None:
            self.vfe_dev = [dict(l, weight=torch.from_numpy(l["weight"]).to(dev)) for l in self.vfe]
            self.vfe_folded = [pe.fold_bn(l["gamma"], l["beta"], l["mean"], l["var"], l["eps"], dev) for l in self.vfe]
            self.se_dev = {k: torch.from_numpy(v).to(dev) for k, v in self.se.items()}
            self.anchors = torch.from_numpy(self.anchors_np).to(dev)
        return self

    def export_numpy(self):
        return dict(self.trunk.export_numpy(), vfe=self.vfe, cam=[cv.np for cv in self.cam_convs], reduc=self.reduc.np,
                    se=self.se, head=self.head.np)

    def fused_image(self):
        Y, X = self.bev_hw
        return torch.empty((Y * X, 2 * self.fuse_C), dtype=torch.float16, device=self.device)

    # ---- stages, device in / device out
    def lidar(self, points, fused, vfe_out=None):
        """points [n, F] (NaN rows are dropped by the voxelizer) -> LiDAR BEV into channels [cam_C, fuse_C) of fused.
        Returns num_voxels [1]."""
        c = self.cfg
        voxels, co, npv, nv = vox.hard_voxelize(points, c["voxel_size"], c["point_cloud_range"], c["max_points"],
                                                c["max_voxels"])
        coors = torch.nn.functional.pad(co, (1, 0))
        feats = pe.hard_vfe(voxels, npv, coors, self.vfe_dev, c["voxel_size"], c["point_cloud_range"], num_voxels=nv,
                            folded=self.vfe_folded, out=vfe_out)
        nx, ny = self.grid
        image, shape = sp.sparse_coo_tensor(coors, feats, [1, 1, ny, nx, self.vfe_C[1]], num=nv).to_pixel_h16()
        self.trunk(image, shape, out=fused, out_channels=self.fuse_C, out_c0=self.cam_C)
        return nv

    def pool(self, depth, feat, prepared, out=None):
        return bp.bev_pool_v2_dev_h16(depth, feat, prepared, self.vt.bev_feat_shape(1), self.pool_C, out=out)

    def camera(self, pool_image, fused):
        """Pool image -> the camera encoder, its last conv into channels [0, cam_C) of fused."""
        Y, X = self.bev_hw
        x, shape = pool_image, (1, Y, X, self.pool_C)
        for cv in self.cam_convs[:-1]:
            x, _, _ = cv(x, shape)
            shape = (1, Y, X, cv.cout)
        self.cam_convs[-1](x, shape, out_h16=fused, out_channels=self.fuse_C, out_c0=0)

    def fuse_and_head(self, fused, gate=None):
        """reduc_conv -> SE gate (in place) -> head conv: planes [1, R (C + 11), Y, X] fp32."""
        Y, X = self.bev_hw
        x, _, _ = self.reduc(fused, (1, Y, X, self.fuse_C))
        fc = self.cfg["fusion_channels"]
        se_gate_h16(x, (1, Y, X, fc), self.se_dev["weight"], self.se_dev["bias"], gate=gate)
        _, planes, _ = self.head(x, (1, Y, X, fc), want_nchw=True)
        return x, planes

    def postprocess(self, planes, out=None):
        t = self.cfg["test"]
        return a3d.anchor3d_postprocess_device(planes, self.anchors, self.num_classes, self.R, t["nms_pre"],
                                               t["score_thr"], t["nms_thr"], t["max_num"], t["dir_offset"],
                                               t["dir_limit_offset"], out=out)

    def forward(self, points, mats, logits, tran_feat):
        """Eager frame: dict of the fused image, the SE output, the head planes and the worst-case-sized decode."""
        fused = self.fused_image()
        nv = self.lidar(points, fused)
        prepared = self.vt.ranks(mats, 1, self.N)
        depth, feat = bp.lss_depth_feat(logits, tran_feat)
        self.camera(self.pool(depth, feat, prepared), fused)
        x, planes = self.fuse_and_head(fused)
        boxes, scores, labels, count = self.postprocess(planes)
        return dict(fused=fused, se=x, planes=planes, boxes=boxes, scores=scores, labels=labels, counts=count,
                    num_voxels=nv)

    def calibrate_cls_bias(self, points, mats, logits, tran_feat, target_frac=0.02):
        """Shift each class's cls biases so that about target_frac / C of the anchors pass score_thr in that class on
        this frame (about 2 % together): more than nms_pre, so the cut runs, and every class reaches the output."""
        planes = self.forward(points, mats, logits, tran_feat)["planes"]
        R, C = self.R, self.num_classes
        cls = planes[0, :R * C].reshape(R, C, -1)
        A = cls.shape[-1] * R
        k = max(1, int(round(target_frac * A / C)))
        thr = self.cfg["test"]["score_thr"]
        logit_thr = float(np.log(thr / (1.0 - thr)))
        b = self.head.np["bias"].copy()
        for c in range(C):
            v = np.sort(cls[:, c].reshape(-1).float().cpu().numpy())[::-1]
            shift = logit_thr - 0.5 * (float(v[k - 1]) + float(v[min(k, len(v) - 1)]))
            b[c:R * C:C] = (b[c:R * C:C] + np.float32(shift)).astype(np.float32)
        self.head.np["bias"] = b
        self.head.dev["shift"].copy_(torch.from_numpy(b))
        return self

    def flops(self):
        """Algorithmic flops (2 x MACs) of the dense convs: camera encoder, LiDAR trunk, reduc_conv, SE gate conv, head."""
        Y, X = self.bev_hw
        out = dict(camera_encoder=sum(2.0 * Y * X * 9 * cv.cin * cv.cout for cv in self.cam_convs), lidar_trunk=0.0)
        h, w = self.grid[1], self.grid[0]
        sizes = []
        for blk in self.trunk.blocks:
            for cv in blk:
                h, w = (h + 2 * cv.padding - cv.k) // cv.stride + 1, (w + 2 * cv.padding - cv.k) // cv.stride + 1
                out["lidar_trunk"] += 2.0 * h * w * cv.cin * cv.cout * cv.k * cv.k
            sizes.append((h, w))
        for (h, w), de in zip(sizes, self.trunk.deblocks):
            out["lidar_trunk"] += 2.0 * (h * de.up) * (w * de.up) * de.cin * de.cout * (1 if de.up > 1 else de.k * de.k)
        fc = self.cfg["fusion_channels"]
        out["fusion"] = 2.0 * Y * X * 9 * self.fuse_C * fc + 2.0 * fc * fc
        out["head"] = 2.0 * Y * X * fc * self.head.cout
        out["total"] = sum(out.values())
        return out


class BEVFusionHotPath(ResultSlotOwner, CameraFrame):
    """One BEVFusion frame as one captured CUDA graph on its own stream: camera descriptor and points H2D; the LiDAR
    branch (voxelize -> HardVFE -> scatter -> trunk into channels [256, 640)) on a forked stream; the camera branch
    (ranks -> softmax / permute -> pool -> encoder into [0, 256)) on the frame stream; the join, reduc_conv, SE gate,
    head conv and anchor3d_postprocess; one D2H through a ResultSlot.  accelerate (the model's view transformer built
    with accelerate=True): the rank graph replays only when the camera matrices change.  Lanes may share one model
    (share_model).  The status word is the device's fp16-pair overflow flag; a cloud larger than the lane's point
    capacity is refused before anything is enqueued."""

    def __init__(self, model, num_points=300000, device="cuda", stream=None):
        super().__init__(model.vt, 1, model.N, device, stream)
        self.model = model
        self.cap = int(num_points)
        self.h_points = torch.full((self.cap, model.F), float("nan"), dtype=torch.float32).pin_memory()
        self.points = torch.full((self.cap, model.F), float("nan"), dtype=torch.float32, device=self.device)
        self.fused = model.fused_image()
        _, Y, X, _ = (1, *model.bev_hw, 0)
        self.pool_image = torch.empty((Y * X, 2 * model.pool_C), dtype=torch.float16, device=self.device)
        self.vfe_out = torch.zeros((model.cfg["max_voxels"], model.vfe_C[1]), dtype=torch.float32, device=self.device)
        self.gate = torch.empty((1, model.cfg["fusion_channels"]), dtype=torch.float32, device=self.device)
        self.side = torch.cuda.Stream(self.device)
        t = model.cfg["test"]
        self.slot = ResultSlot(t["max_num"], 9, 1, 1)

    def share_model(self, other):
        self.model, self.vt = other.model, other.vt
        return self

    def _frame(self):
        m = self.model
        main = torch.cuda.current_stream(self.device)
        self.side.wait_stream(main)
        with torch.cuda.stream(self.side):
            self.points.copy_(self.h_points, non_blocking=True)
            nv = m.lidar(self.points, self.fused, vfe_out=self.vfe_out)
        bp.lss_depth_feat(self.logits, self.tran_feat, self.depth, self.feat)
        m.pool(self.depth, self.feat, self.prepared, out=self.pool_image)
        m.camera(self.pool_image, self.fused)
        main.wait_stream(self.side)
        x, planes = m.fuse_and_head(self.fused, gate=self.gate)
        boxes, scores, labels, count = m.postprocess(planes)
        out = dict(boxes=boxes, scores=scores, labels=labels, counts=count, status=sp.status_tensor(self.device),
                   planes=planes, se=x, num_voxels=nv)
        self.slot.copy_from(out)
        return out

    def launch(self, points, mats, logits=None, tran_feat=None):
        """Enqueue one frame: points [n, F] host array or tensor (n <= the lane's capacity, else ValueError before
        anything is enqueued), mats = (sensor2ego, cam2imgs, post_rots, post_trans, bda) on the host, logits / tran_feat
        device tensors (None: already in the frame's inputs)."""
        pts = torch.as_tensor(np.asarray(points, np.float32) if not isinstance(points, torch.Tensor) else points)
        if pts.dim() != 2 or pts.shape[1] != self.model.F:
            raise ValueError("points must be [n, %d]" % self.model.F)
        if pts.shape[0] > self.cap:
            raise ValueError("BEVFusion: %d points exceed the lane's capacity of %d" % (pts.shape[0], self.cap))

        def host_inputs():
            n = pts.shape[0]
            self.h_points[:n].copy_(pts)
            self.h_points[n:].fill_(float("nan"))
        self._launch(mats, logits, tran_feat, "frame", host_inputs)

    def result(self):
        """Wait for the last launched frame: (boxes [K, 9], scores [K], labels [K]) host tensors owned by the lane."""
        return self.slot.read(self.check_status, self.done)

    def infer(self, points, mats, logits=None, tran_feat=None):
        self.launch(points, mats, logits, tran_feat)
        return self.result()

    def infer_many(self, items):
        """items: (points, mats, logits, tran_feat) tuples, one frame each, waited for one by one; the results cloned."""
        out = []
        for it in items:
            self.launch(*it)
            out.append(tuple(t.clone() for t in self.result()))
        return out

    def check_status(self, status_host):
        if int(status_host[0]):
            raise RuntimeError("BEVFusion: an activation left fp16's range (|x| >= 65504) on the fp16-pair path")
