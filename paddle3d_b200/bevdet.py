"""BEVDet inference on one GPU from the depth net's output on (BEVDet-R50's BEV half, PARITY UNPINNED: the model values in
CONFIG are recalled from BEVDet's bevdet-r50 config, which Paddle3D's configs/bevdet descend from; they were not checked
against either file):

    camera descriptor H2D -> p3d_lss_prepare -> depth softmax / permute -> bev_pool straight into the pixel fp16-pair image
    [128 x 128 x 96] (channels 80..95 zero) -> CustomResNet (BasicBlocks, residual added in the conv epilogue) -> FPN_LSS
    (bilinear x4 / x2 with align_corners on the pair rows) -> CenterHead (dense_head.DenseRPNHead with this encoder as its
    trunk) -> centerpoint_postprocess_device or bevdet_postprocess_device -> boxes

BEVDetHotPath captures all of it, from the descriptor upload to the D2H copy of the boxes, as one CUDA graph.  Which
decode runs follows from the model's test config, as in the reference's configs: one without nms_type (CONFIG) runs the
custom op Paddle3D's predict_by_custom_op calls (arg-max class per cell, one rotated NMS threshold, 83 boxes per task,
gravity centre); one with nms_type (CONFIG_BEVDET_NMS) runs BEVDet's own get_bboxes (ops.bevdet_postprocess: top-K over
class x cell, per-class scale-NMS or circle NMS, bottom centre, up to post_max_size boxes per task).

BEVDetFromImages / BEVDetImageHotPath (CONFIG_IMG) put BEVDet's image half in front of it: six normalised camera images ->
ResNet-50 (p3d_resnet_stem_h16, then Bottlenecks on the dense fp16-pair conv) -> CustomFPN -> depth net ->
p3d_lss_depth_feat_h16 -> the frame above, one captured graph.

BEVDetFrameHotPath (DATA_CONFIG) starts that graph one step earlier, from six decoded uint8 camera frames: the test
pipeline's resize, crop and normalisation (ops.image_prep, bit-identical to Pillow + OpenCV on the host) -> the images.

BEVDet4DFromImages / BEVDet4DImageHotPath / BEVDet4DFrameHotPath (CONFIG_4D_IMG) do the same for BEVDet4D: the image
encoder (and the image prep) at the head of both temporal graphs; BEVDet4DFrameHotPath.infer_stream runs a drive from
frames and ego poses (drive_mats)."""
import functools
import itertools

import numpy as np
import torch

from . import raw, synth
from .dense_head import DenseRPNHead, _Conv
from .frame import ResultSlot, ResultSlotOwner, StagedUpload, copy_rows, in_flight
from .lss import CameraFrame, LSSViewTransformer
from .ops import bev_pool_v2 as bp
from .ops import bevdet_postprocess as bdp
from .ops import centerpoint_postprocess as cpp
from .ops import dense_conv as dc
from .ops import image_prep as ip
from .ops import jpeg
from .ops import sparse_nn as sp

# PARITY UNPINNED (see the module docstring)
CONFIG = dict(
    grid=synth.LSS_BEVDET, input_size=synth.LSS_INPUT_SIZE, downsample=synth.LSS_DOWNSAMPLE, channels=synth.LSS_CHANNELS,
    n_cams=6,
    backbone=dict(num_channels=(160, 320, 640), strides=(2, 2, 2), blocks=2, bn_eps=1e-5),
    fpn=dict(in_channels=800, out_channels=256, scale_factor=4, input_feature_index=(0, 2), extra_upsample=2, bn_eps=1e-5),
    head=dict(tasks=tuple(synth.CENTERPOINT_TASKS), share_conv_channel=64),
    # voxel size 0.1 x down_ratio 8 = the 0.8 m cells of the BEV grid
    test=dict(synth.CENTERPOINT_TEST_CFG, voxel_size=(0.1, 0.1), point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]),
)

# PARITY UNPINNED: BEVDet's own test config, recalled from bevdet-r50 (tasks: car | truck, construction vehicle | bus,
# trailer | barrier | motorcycle, bicycle | pedestrian, traffic cone).  nms_rescale_factor is per task a scalar or one
# factor per class; max_per_img is carried for completeness: get_bboxes never reads it.
TEST_CFG_BEVDET = dict(
    max_num=500, score_threshold=0.1, out_size_factor=8, pre_max_size=1000, post_max_size=500, max_per_img=500,
    post_center_limit_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0],
    nms_type=["rotate", "rotate", "rotate", "circle", "rotate", "rotate"],
    nms_thr=[0.2, 0.2, 0.2, 0.2, 0.2, 0.5],
    nms_rescale_factor=[1.0, [0.7, 0.7], [0.4, 0.55], 1.1, [1.0, 1.0], [4.5, 9.0]],
    min_radius=[4, 12, 10, 1, 0.85, 0.175],
    voxel_size=(0.1, 0.1), point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0])
CONFIG_BEVDET_NMS = dict(CONFIG, test=TEST_CFG_BEVDET)


def round32(c):
    return (int(c) + 31) // 32 * 32


class BEVDetEncoder:
    """CustomResNet (BasicBlocks: relu(bn2(conv2(relu(bn1(conv1(x))))) + identity); the first block of a stage has a 3x3
    stride-s conv1 and a 3x3 stride-s Conv2d with bias as its identity branch) + FPN_LSS (cat([x0, up4(x2)]), two 3x3
    ConvModules, up2, a 3x3 ConvModule and a 1x1 conv with bias), on pixel fp16-pair rows.  A DenseRPNHead trunk.
    in_pad: channels of the input image rows (the pool image's, in_channels rounded up to 32); the first stage's weights
    are zero-padded on Cin to it once, when they are packed."""

    def __init__(self, in_channels, num_channels, strides, blocks, fpn_out, scale_factor=None, input_feature_index=None,
                 extra_upsample=None, bn_eps=1e-5, in_pad=None, row_pad=None):
        """fpn_out None: CustomResNet alone (BEVDet4D's pre_process net).  row_pad: channels of the rows every conv writes
        (None: its Cout); every conv's weights are zero-padded on Cin to the rows it reads, whose padding channels the
        caller keeps zero (pre_process writes 80 channels into 96-channel rows)."""
        self.in_channels, self.in_pad = in_channels, in_pad or round32(in_channels)
        self.row_pad = row_pad
        self.scale_factor, self.extra_upsample = scale_factor, extra_upsample
        self.stages = []
        cin, rows = in_channels, self.in_pad
        for cout, s in zip(num_channels, strides):
            out_rows = row_pad or cout
            pad = rows if rows != cin else None
            rpad = out_rows if out_rows != cout else None
            stage = [dict(conv1=_Conv(cin, cout, 3, s, 1, bn_eps=bn_eps, cin_pad=pad),
                          conv2=_Conv(cout, cout, 3, 1, 1, bn_eps=bn_eps, cin_pad=rpad),  # ReLU after the residual
                          down=_Conv(cin, cout, 3, s, 1, bias=True, relu=False, cin_pad=pad))]
            for _ in range(blocks - 1):
                stage.append(dict(conv1=_Conv(cout, cout, 3, 1, 1, bn_eps=bn_eps, cin_pad=rpad),
                                  conv2=_Conv(cout, cout, 3, 1, 1, bn_eps=bn_eps, cin_pad=rpad), down=None))
            self.stages.append(stage)
            cin, rows = cout, out_rows
        self.stage_channels = tuple(num_channels)
        self.fpn, self.fpn_channels, self.index, self.cat_channels = [], None, None, None
        if fpn_out is None:
            return
        self.index = tuple(input_feature_index)
        self.cat_channels = num_channels[self.index[0]] + num_channels[self.index[1]]
        mid = fpn_out * (2 if extra_upsample else 1)
        self.fpn = [_Conv(self.cat_channels, mid, 3, 1, 1, bn_eps=bn_eps), _Conv(mid, mid, 3, 1, 1, bn_eps=bn_eps),
                    _Conv(mid, fpn_out, 3, 1, 1, bn_eps=bn_eps), _Conv(fpn_out, fpn_out, 1, 1, 0, bias=True, relu=False)]
        self.fpn_channels = fpn_out

    def convs(self):
        out = []
        for stage in self.stages:
            for blk in stage:
                out += [blk["conv1"], blk["conv2"]] + ([blk["down"]] if blk["down"] is not None else [])
        return out + list(self.fpn)

    def export_numpy(self):
        return dict(backbone=[[{k: (c.np if c is not None else None) for k, c in blk.items()} for blk in stage]
                              for stage in self.stages],
                    fpn=[c.np for c in self.fpn], fpn_index=self.index, scale_factor=self.scale_factor,
                    extra_upsample=self.extra_upsample)

    def _block(self, blk, x, shape, bufs=None, out=None):
        """One BasicBlock.  bufs: dict conv name -> preallocated output rows (None / missing: allocated); out = (rows,
        channels, c0): conv2 writes channels [c0, c0 + Cout) of those rows instead."""
        b = shape[0]
        bufs = bufs or {}
        cout = blk["conv1"].cout
        rows = self.row_pad or cout
        t, _, (_, oh, ow) = blk["conv1"](x, shape, out_h16=bufs.get("conv1"), out_channels=rows)
        idn = x if blk["down"] is None else blk["down"](x, shape, out_h16=bufs.get("down"), out_channels=rows)[0]
        o, oc, c0 = out or (bufs.get("conv2"), rows, 0)
        y, _, _ = blk["conv2"](t, (b, oh, ow, rows), residual=idn, res_channels=rows, out_h16=o, out_channels=oc, out_c0=c0)
        return y, (b, oh, ow, rows)

    def backbone(self, x, shape, bufs=None, out=None):
        """CustomResNet: the pixel image of every stage's output, [(rows, (B, H, W, C))].  bufs: per stage, per block, the
        _block buffers; out: where the last conv writes (_block)."""
        feats = []
        for si, stage in enumerate(self.stages):
            for bi, blk in enumerate(stage):
                last = si == len(self.stages) - 1 and bi == len(stage) - 1
                x, shape = self._block(blk, x, shape, bufs[si][bi] if bufs else None, out if last else None)
            feats.append((x, shape))
        return feats

    def __call__(self, x, shape, first=None):
        """x: pixel fp16-pair rows [B*H*W, 2*in_pad], shape = (B, H, W, in_pad).  Returns (FPN_LSS output rows, shape)."""
        if first is not None or int(shape[3]) != self.in_pad or not self.fpn:
            raise ValueError("BEVDetEncoder takes the %d-channel pool image" % self.in_pad)
        feats = self.backbone(x, shape)
        (x0, s0), (x2, s2) = feats[self.index[0]], feats[self.index[1]]
        b, h, w, c0 = s0
        cat_c = self.cat_channels
        cat = torch.empty((b * h * w, 2 * cat_c), dtype=torch.float16, device=x.device)
        dc.upsample_bilinear_h16(x0, s0, 1, out_h16=cat, out_channels=cat_c, out_c0=0)
        dc.upsample_bilinear_h16(x2, s2, self.scale_factor, out_h16=cat, out_channels=cat_c, out_c0=c0)
        f0, f1, f2, f3 = self.fpn
        y, _, _ = f0(cat, (b, h, w, cat_c))
        y, _, _ = f1(y, (b, h, w, f0.cout))
        if self.extra_upsample:
            y, (b, h, w) = dc.upsample_bilinear_h16(y, (b, h, w, f1.cout), self.extra_upsample)
        y, _, _ = f2(y, (b, h, w, f1.cout))
        y, _, _ = f3(y, (b, h, w, f2.cout))
        return y, (b, h, w, f3.cout)


class BEVDet:
    """Seeded BEVDet (CONFIG) from the depth net's output: LSSViewTransformer, BEVDetEncoder and the CenterHead.  Batch 1
    (the postprocess is batch 1)."""

    def __init__(self, model_cfg=None, accelerate=False, device="cuda"):
        self.mc = mc = model_cfg or CONFIG
        self.device = torch.device(device)
        self.N = mc["n_cams"]
        self.vt = LSSViewTransformer(mc["grid"], mc["input_size"], mc["downsample"], mc["channels"], accelerate=accelerate,
                                     device=self.device)
        X, Y, Z = self.vt.grid
        self.pool_C = round32(Z * mc["channels"])
        b, f, h = mc["backbone"], mc["fpn"], mc["head"]
        enc_in = b.get("in_channels", Z * mc["channels"])  # BEVDet4D: the 160-channel concat
        self.encoder = BEVDetEncoder(enc_in, b["num_channels"], b["strides"], b["blocks"], f["out_channels"],
                                     f["scale_factor"], f["input_feature_index"], f["extra_upsample"], b["bn_eps"],
                                     round32(enc_in))
        if self.encoder.cat_channels != f["in_channels"]:
            raise ValueError("FPN_LSS in_channels %d, the concat has %d" % (f["in_channels"], self.encoder.cat_channels))
        self.head = DenseRPNHead(in_channels=f["out_channels"], tasks=h["tasks"], share_conv_channel=h["share_conv_channel"],
                                 bev_depth=1, trunk=self.encoder)
        self.test_cfg = dict(mc["test"])
        self.label_off = synth.label_offsets(list(h["tasks"]))
        self.image_shape = (1, Y, X, self.pool_C)
        self.enc_shape = (1, Y, X, self.encoder.in_pad)  # the encoder's input rows (BEVDet: the pool image)

    def init_weight(self, seed=0, bn_gain=1.0, device=None):
        """Seeded weights (dense_head.DenseRPNHead.init_weight); device=False: numpy parameters only."""
        self.head.init_weight(seed=seed, device=None if device is False else (device or self.device), bn_gain=bn_gain)
        return self

    def export_numpy(self):
        return self.head.export_numpy()

    # ---- stages, device in / device out
    def pool(self, depth, feat, prepared, out=None):
        """bev_pool into the pixel fp16-pair image [Y*X, 2*pool_C]."""
        return bp.bev_pool_v2_dev_h16(depth, feat, prepared, self.vt.bev_feat_shape(1), self.pool_C, out=out)

    def image(self, mats, logits, tran_feat):
        """Eager view transform into the pool image: mats = (sensor2ego, cam2imgs, post_rots, post_trans, bda)."""
        prepared = self.vt.ranks(mats, 1, self.N)
        depth, feat = bp.lss_depth_feat(logits, tran_feat)
        return self.pool(depth, feat, prepared)

    def encode(self, image):
        return self.encoder(image, self.enc_shape)

    def dense(self, image):
        """Encoder input (BEVDet: the pool image) -> dict name -> per-task [1, k, 128, 128] fp32 head planes."""
        return self.head.forward_h16(image, self.enc_shape)

    def result_rows(self):
        """Rows of the worst-case-sized outputs of postprocess."""
        tc = self.test_cfg
        return len(self.label_off) * tc["post_max_size" if "nms_type" in tc else "nms_post_max_size"]

    def postprocess(self, h):
        tc = self.test_cfg
        if "nms_type" in tc:  # BEVDet's get_bboxes; without it the Paddle custom op's rules
            return bdp.bevdet_postprocess_heads(h, tc, self.label_off)
        return cpp.centerpoint_postprocess_heads(h, tc["voxel_size"], tc["point_cloud_range"], tc, self.label_off)

    def forward(self, mats, logits, tran_feat):
        """Eager frame: (boxes, scores, labels, counts) on the device, worst-case sized (counts[-1] rows valid)."""
        return self.postprocess(self.dense(self.image(mats, logits, tran_feat)))

    def calibrate_heatmap_bias(self, mats, logits, tran_feat, target_frac=0.014):
        """DenseRPNHead.calibrate_heatmap_bias on this frame: ~1.4 % of the cells above the score threshold, as the LiDAR
        frames do.  Weights stay seeded and are exported unchanged to the CPU arm."""
        img = self.image(mats, logits, tran_feat)
        self.head.calibrate_heatmap_bias(img, self.test_cfg["score_threshold"], target_frac, shape=self.enc_shape)
        return self

    def flops(self):
        """Algorithmic flops (2 x MACs) of the dense part: backbone (CustomResNet with its identity convs), FPN_LSS and
        the head (shared conv, the 36 ConvModules, the output convs).  The Cin padding 80 -> 96 is not counted."""
        out = dict(backbone=0.0, fpn=0.0)
        _, H, W, _ = self.image_shape
        h, w = H, W
        for stage in self.encoder.stages:
            for blk in stage:
                c1 = blk["conv1"]
                h, w = (h + 2 * c1.padding - c1.k) // c1.stride + 1, (w + 2 * c1.padding - c1.k) // c1.stride + 1
                for c in blk.values():
                    if c is not None:
                        out["backbone"] += 2.0 * h * w * c.cin * c.cout * c.k * c.k
        enc = self.encoder
        s0 = enc.stages[enc.index[0]][0]["conv1"].stride
        h0 = H // s0  # x0's size (the concat's)
        h1 = h0 * (enc.extra_upsample or 1)
        f0, f1, f2, f3 = enc.fpn
        for c, hh in ((f0, h0), (f1, h0), (f2, h1), (f3, h1)):
            out["fpn"] += 2.0 * hh * hh * c.cin * c.cout * c.k * c.k
        out.update(self.head.head_flops(h1, h1))
        out["total"] = out["backbone"] + out["fpn"] + out["head"]
        return out

    def head_planes(self):
        return self.head.head_planes()


class BEVDetHotPath(ResultSlotOwner, CameraFrame):
    """One BEVDet frame as one captured CUDA graph on its own stream (CameraFrame): camera descriptor H2D ->
    p3d_lss_prepare -> depth softmax / permute -> memset + pool into the pixel image -> encoder -> head -> postprocess ->
    one D2H of boxes [6 x 83, 9] ([6 x 500, 9] with BEVDet's own decode), scores, labels, counts and the status word.  Any calibration replays the same graph.
    accelerate (the model's view transformer built with accelerate=True): two graphs, ranks (replayed only when the camera
    matrices differ from the last ones) and the rest.  Several lanes may share one model (share_model), each with its own
    buffers and stream.  The status word is the device's fp16-pair overflow flag (ops.sparse_nn.status_tensor), which
    stays set once raised."""

    def __init__(self, model, device="cuda", stream=None):
        super().__init__(model.vt, 1, model.N, device, stream)
        self.model = model
        _, Y, X, pc = model.image_shape
        self.image = torch.empty((Y * X, 2 * pc), dtype=torch.float16, device=self.device)
        self.slot = ResultSlot(model.result_rows(), 9, len(model.label_off) + 1, 1)

    def share_model(self, other):
        self.model, self.vt = other.model, other.vt
        return self

    # ---- stages, as they are captured
    def _depth_feat(self):
        """The frame's first stage: fill self.depth / self.feat (here from the depth net's output in self.logits /
        self.tran_feat; ImageInput and FrameInput override it)."""
        bp.lss_depth_feat(self.logits, self.tran_feat, self.depth, self.feat)

    def _frame(self):
        self._depth_feat()
        self.model.pool(self.depth, self.feat, self.prepared, out=self.image)
        return self._dense(self.image)

    def _dense(self, x):
        """Encoder -> head -> postprocess from the encoder's input rows x, then the D2H copies."""
        m = self.model
        h = m.dense(x)
        boxes, scores, labels, counts = m.postprocess(h)
        out = dict(boxes=boxes, scores=scores, labels=labels, counts=counts, status=sp.status_tensor(self.device), head=h)
        self.slot.copy_from(out)
        return out

    def result(self):
        """Wait for the last launched frame: (boxes [K, 9], scores [K], labels [K]) host tensors owned by the lane (valid
        until its next launch); raises from check_status."""
        return self.slot.read(self.check_status, self.done)

    def infer(self, mats, logits=None, tran_feat=None):
        self.launch(mats, logits, tran_feat)
        return self.result()

    def check_status(self, status_host):
        """Raise when an activation left fp16's range on the fp16-pair path (never a silent wrong result)."""
        if int(status_host[0]):
            raise RuntimeError("BEVDet: an activation left fp16's range (|x| >= 65504) on the fp16-pair path")


# ------------------------------------------------------------------------------------------------ BEVDet from images
# PARITY UNPINNED, as CONFIG: BEVDet-R50's image half, recalled from bevdet-r50 (not checked against it or Paddle3D's
# configs/bevdet): img_backbone = mmdet ResNet(depth=50, num_stages=4, out_indices=(2, 3), style='pytorch') with BN (eval,
# eps 1e-5); img_neck = CustomFPN(in_channels=[1024, 2048], out_channels=512, num_outs=1, start_level=0, out_ids=[0]);
# the view transformer's depth_net = Conv2d(512, D + C, 1).  Stages: (planes, blocks, stride).
IMG_BACKBONE = dict(depth=50, stages=((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)), out_indices=(2, 3), bn_eps=1e-5)
IMG_NECK = dict(in_channels=(1024, 2048), out_channels=512)
DEPTH_NET = dict(in_channels=512)
CONFIG_IMG = dict(CONFIG, img_backbone=IMG_BACKBONE, img_neck=IMG_NECK, depth_net=DEPTH_NET)
CONFIG_IMG_BEVDET_NMS = dict(CONFIG_IMG, test=TEST_CFG_BEVDET)

# PARITY UNPINNED, as CONFIG: bevdet-r50's data_config as its test pipeline reads it (PrepareImageInputs with
# train=False: resize to input_size's width, crop the bottom rows, no flip or rotation) and mmlabNormalize's mean / std
# (float32 arrays there, to_rgb=True), recalled, not checked against the reference.  A model config without data_config
# takes this one at its own input_size.
DATA_CONFIG = dict(src_size=(900, 1600), input_size=(256, 704), crop_h=(0.0, 0.0), resize_test=0.0,
                   mean=(123.675, 116.28, 103.53), std=(58.395, 57.12, 57.375), to_rgb=True)


def round16(c):
    return (int(c) + 15) // 16 * 16


class BEVDetImageEncoder:
    """BEVDet's image encoder on pixel fp16-pair rows: ResNet-50 (stem: p3d_resnet_stem_h16, conv 7x7 s2 + BN + ReLU +
    MaxPool 3x3 s2 in one kernel; Bottlenecks relu(bn3(conv3(relu(bn2(conv2(relu(bn1(conv1(x))))))) + identity), the
    stride on the 3x3 conv, a 1x1 stride-s conv + BN as the identity of each stage's first block, the add in conv3's
    epilogue), CustomFPN on stages 2 and 3 (1x1 lateral convs with bias; lateral1 nearest-upsampled x2 into the residual
    rows of lateral0's conv, so the top-down add happens in its epilogue; a 3x3 conv with bias) and the depth net (1x1
    conv 512 -> D + C with bias, computed as round16(D + C) channels into round32 rows, the extra ones zero).

    Seeded weights (init_weight) stay inside fp16's range: _Conv's uniform init scales a signal's mean square by ~1/3
    and ReLU halves it, so the BN gains are sqrt(6) after a ReLU-ed conv (STEM_GAIN, MID_GAIN), sqrt(3) on the downsample
    identity (DOWN_GAIN), and RES_GAIN on each Bottleneck's last BN (zero_init_residual in spirit: the residual stream of
    the 16 blocks grows slowly).  Per-stage max |x| of the seeded model (seed 0) on synth.camera_images at 256 x 704, six
    cameras (fp64): stem 12.5, layer1 12.9, layer2 11.4, layer3 7.6, layer4 6.2, CustomFPN 1.6, depth net 1.1."""

    STEM_GAIN = MID_GAIN = 6.0 ** 0.5
    DOWN_GAIN = 3.0 ** 0.5
    RES_GAIN = 0.5

    def __init__(self, backbone, neck, depth_net, D, C):
        eps = backbone["bn_eps"]
        self.D, self.C = int(D), int(C)
        self.stem = _Conv(3, 64, 7, 2, 3, bn_eps=eps)  # runs on p3d_resnet_stem_h16, not the dense conv
        self.stages, cin = [], 64
        for planes, blocks, stride in backbone["stages"]:
            stage = []
            for bi in range(blocks):
                s = stride if bi == 0 else 1
                stage.append(dict(conv1=_Conv(cin, planes, 1, 1, 0, bn_eps=eps),
                                  conv2=_Conv(planes, planes, 3, s, 1, bn_eps=eps),
                                  conv3=_Conv(planes, 4 * planes, 1, 1, 0, bn_eps=eps),  # ReLU after the residual
                                  down=_Conv(cin, 4 * planes, 1, s, 0, bn_eps=eps, relu=False) if bi == 0 else None))
                cin = 4 * planes
            self.stages.append(stage)
        self.out_indices = tuple(backbone["out_indices"])
        c0, c1 = neck["in_channels"]
        if (c0, c1) != tuple(4 * self.stages[i][0]["conv1"].cout for i in self.out_indices):
            raise ValueError("CustomFPN in_channels %s do not match the ResNet's stages %s" % ((c0, c1), self.out_indices))
        oc = neck["out_channels"]
        self.lateral = [_Conv(c0, oc, 1, 1, 0, bias=True, relu=False), _Conv(c1, oc, 1, 1, 0, bias=True, relu=False)]
        self.fpn_conv = _Conv(oc, oc, 3, 1, 1, bias=True, relu=False)
        if depth_net["in_channels"] != oc:
            raise ValueError("depth_net in_channels %d, the neck gives %d" % (depth_net["in_channels"], oc))
        self.out_C = round32(self.D + self.C)  # the depth net's rows
        self.depth_net = _Conv(oc, self.D + self.C, 1, 1, 0, bias=True, relu=False, cout_pad=round16(self.D + self.C))
        self.stem_dev = None

    def convs(self):
        """Every conv in parameter order (the stem first)."""
        out = [self.stem]
        for stage in self.stages:
            for blk in stage:
                out += [blk["conv1"], blk["conv2"], blk["conv3"]] + ([blk["down"]] if blk["down"] is not None else [])
        return out + self.lateral + [self.fpn_conv, self.depth_net]

    def init_weight(self, seed=0, device=None):
        """Seeded parameters (numpy; with a device also the packed device images).  Gains: see the class docstring."""
        rng = np.random.default_rng([seed, 6])
        self.stem.init(rng, None, bn_gain=self.STEM_GAIN)
        for stage in self.stages:
            for blk in stage:
                blk["conv1"].init(rng, device, bn_gain=self.MID_GAIN)
                blk["conv2"].init(rng, device, bn_gain=self.MID_GAIN)
                blk["conv3"].init(rng, device, bn_gain=self.RES_GAIN)
                if blk["down"] is not None:
                    blk["down"].init(rng, device, bn_gain=self.DOWN_GAIN)
        for c in self.lateral + [self.fpn_conv, self.depth_net]:
            c.init(rng, device)
        if device is not None:
            p = self.stem.np
            bn = p["bn"]
            sc = bn["gamma"].astype(np.float64) / np.sqrt(bn["var"].astype(np.float64) + bn["eps"])
            sh = -bn["mean"].astype(np.float64) * sc + bn["beta"]
            self.stem_dev = dict(packed=dc.pack_stem_weight(torch.from_numpy(p["weight"]).to(device)),
                                 scale=torch.from_numpy(sc.astype(np.float32)).to(device),
                                 shift=torch.from_numpy(sh.astype(np.float32)).to(device))
        return self

    def export_numpy(self):
        return dict(stem=self.stem.np,
                    stages=[[{k: (c.np if c is not None else None) for k, c in blk.items()} for blk in stage]
                            for stage in self.stages],
                    out_indices=self.out_indices, lateral=[c.np for c in self.lateral], fpn_conv=self.fpn_conv.np,
                    depth_net=self.depth_net.np, D=self.D, C=self.C)

    # ---- device stages (pixel fp16-pair rows in and out)
    def stem_forward(self, imgs):
        d = self.stem_dev
        return dc.resnet_stem_h16(imgs, d["packed"], d["scale"], d["shift"])

    @staticmethod
    def bottleneck(blk, x, shape):
        """One Bottleneck: (rows, (B, oH, oW, 4 planes))."""
        b = shape[0]
        t, _, _ = blk["conv1"](x, shape)
        t, _, (_, oh, ow) = blk["conv2"](t, (b, shape[1], shape[2], blk["conv1"].cout))
        c3 = blk["conv3"]
        idn = x if blk["down"] is None else blk["down"](x, shape)[0]
        y, _, _ = c3(t, (b, oh, ow, blk["conv2"].cout), residual=idn, res_channels=c3.cout)
        return y, (b, oh, ow, c3.cout)

    def stage_forward(self, si, x, shape):
        for blk in self.stages[si]:
            x, shape = self.bottleneck(blk, x, shape)
        return x, shape

    def backbone(self, imgs):
        """The pixel rows of every stage's output after the stem, [(rows, (B, H, W, C))]."""
        x, shape = self.stem_forward(imgs)
        feats = []
        for si in range(len(self.stages)):
            x, shape = self.stage_forward(si, x, shape)
            feats.append((x, shape))
        return feats

    def neck(self, feats):
        """CustomFPN: (rows, shape) of its 512-channel output."""
        (x0, s0), (x1, s1) = feats[self.out_indices[0]], feats[self.out_indices[1]]
        l0c, l1c = self.lateral
        oc = l0c.cout
        l1, _, _ = l1c(x1, s1)
        up, (b, h, w) = dc.upsample_nearest_h16(l1, (s1[0], s1[1], s1[2], oc), s0[1] // s1[1])
        if (h, w) != tuple(s0[1:3]):
            raise ValueError("CustomFPN: lateral1 %s does not upsample to lateral0 %s" % ((h, w), tuple(s0[1:3])))
        l0, _, _ = l0c(x0, s0, residual=up, res_channels=oc)
        y, _, _ = self.fpn_conv(l0, (b, h, w, oc))
        return y, (b, h, w, oc)

    def head(self, y, shape):
        """The depth net: rows [B*H*W, 2*out_C] (channels [0, D) logits, [D, D + C) tran_feat, the rest zero)."""
        b, h, w, _ = shape
        out = torch.zeros((b * h * w, 2 * self.out_C), dtype=torch.float16, device=y.device) \
            if self.out_C > self.depth_net.cout_pad else None
        d, _, _ = self.depth_net(y, shape, out_h16=out, out_channels=self.out_C)
        return d, (b, h, w, self.out_C)

    def __call__(self, imgs):
        """imgs [N, 3, H, W] fp32 (normalised) -> the depth net's pixel rows and their shape (N, H / 16, W / 16, out_C)."""
        return self.head(*self.neck(self.backbone(imgs)))

    def flops(self, H, W, n):
        """Algorithmic flops (2 x MACs) of n images at H x W: stem, layers, neck, depth net (D + C outputs, unpadded)."""
        ch, cw = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        out = dict(img_stem=2.0 * n * ch * cw * 3 * 49 * 64)
        h, w = dc.stem_shape(H, W)
        layers, sizes = 0.0, []
        for stage in self.stages:
            for blk in stage:
                s = blk["conv2"].stride
                oh, ow = (h - 1) // s + 1, (w - 1) // s + 1
                layers += 2.0 * n * (h * w * blk["conv1"].cin * blk["conv1"].cout
                                     + oh * ow * 9 * blk["conv2"].cin * blk["conv2"].cout
                                     + oh * ow * blk["conv3"].cin * blk["conv3"].cout)
                if blk["down"] is not None:
                    layers += 2.0 * n * oh * ow * blk["down"].cin * blk["down"].cout
                h, w = oh, ow
            sizes.append((h, w))
        out["img_layers"] = layers
        out["img_backbone"] = out["img_stem"] + layers
        (h0, w0), (h1, w1) = sizes[self.out_indices[0]], sizes[self.out_indices[1]]
        l0, l1, f = self.lateral[0], self.lateral[1], self.fpn_conv
        out["img_neck"] = 2.0 * n * (h0 * w0 * l0.cin * l0.cout + h1 * w1 * l1.cin * l1.cout + h0 * w0 * 9 * f.cin * f.cout)
        out["depth_net"] = 2.0 * n * h0 * w0 * self.depth_net.cin * self.depth_net.cout
        return out


class BEVDetFromImages(BEVDet):
    """BEVDet (CONFIG_IMG) from six normalised camera images: BEVDetImageEncoder, p3d_lss_depth_feat_h16 on its rows, then
    BEVDet's view transform, encoder, head and postprocess.  Batch 1.  input_size must be a multiple of 32 (so that the
    ResNet's stride-16 stage is input_size // 16 and CustomFPN's x2 upsampling is exact)."""

    def __init__(self, model_cfg=None, accelerate=False, device="cuda"):
        mc = model_cfg or CONFIG_IMG
        H_in, W_in = mc["input_size"]
        if H_in % 32 or W_in % 32:
            raise ValueError("BEVDetFromImages: input_size %s is not a multiple of 32" % (tuple(mc["input_size"]),))
        if mc["downsample"] != 16:
            raise ValueError("BEVDetFromImages: the depth net runs on the ResNet's stride-16 stage (downsample 16), got %r"
                             % mc["downsample"])
        super().__init__(mc, accelerate, device)
        self.input_size = (int(H_in), int(W_in))
        self.image_encoder = BEVDetImageEncoder(mc["img_backbone"], mc["img_neck"], mc["depth_net"], self.vt.D,
                                                mc["channels"])
        self.data_config = dict(mc.get("data_config", dict(DATA_CONFIG, input_size=self.input_size)))
        self.augmentation = ip.test_augmentation(self.data_config)
        x0, y0, x1, y1 = self.augmentation["crop"]
        if (y1 - y0, x1 - x0) != self.input_size:
            raise ValueError("BEVDetFromImages: data_config crops %s images, the model takes %s"
                             % ((y1 - y0, x1 - x0), self.input_size))
        self.prep_plan = None

    def init_weight(self, seed=0, bn_gain=1.0, device=None):
        """Seeded weights; with a device also the image prep plan of data_config (ops.image_prep.ImagePrepPlan)."""
        super().init_weight(seed=seed, bn_gain=bn_gain, device=device)
        self.image_encoder.init_weight(seed, device=None if device is False else (device or self.device))
        if device is not False:
            self.prep_plan = ip.ImagePrepPlan.from_data_config(self.data_config, device or self.device)
        return self

    def test_mats(self, sensor2ego, cam2imgs, bda):
        """(sensor2ego, cam2imgs, post_rots, post_trans, bda) of camera frames run through data_config's test
        augmentation: post_rots / post_trans [B, N, 3, 3] / [B, N, 3] float32 from it."""
        b, n = np.shape(sensor2ego)[:2]
        a = self.augmentation
        return (sensor2ego, cam2imgs, np.broadcast_to(a["post_rot"], (b, n, 3, 3)).copy(),
                np.broadcast_to(a["post_tran"], (b, n, 3)).copy(), bda)

    def images_from_frames(self, frames):
        """frames [N, H0, W0, 3] uint8 on the device (decoded RGB) -> the normalised images [N, 3, H, W] fp32."""
        if self.prep_plan is None:
            raise RuntimeError("BEVDetFromImages: call init_weight with a device first (it builds the image prep plan)")
        return ip.image_prep_u8(frames, self.prep_plan)

    def forward_frames(self, sensor2ego, cam2imgs, bda, frames):
        """Eager frame from decoded camera frames [N, H0, W0, 3] uint8 on the device: (boxes, scores, labels, counts) as
        forward_images on images_from_frames(frames) with test_mats."""
        return self.forward_images(self.test_mats(sensor2ego, cam2imgs, bda), self.images_from_frames(frames))

    def export_numpy(self):
        return dict(super().export_numpy(), image_encoder=self.image_encoder.export_numpy())

    def stage_shapes(self):
        """(C, H, W) of the stem and of every ResNet stage's output, then of the depth net's rows."""
        H, W = self.input_size
        h, w = dc.stem_shape(H, W)
        out = [(64, h, w)]
        for stage in self.image_encoder.stages:
            s = stage[0]["conv2"].stride
            h, w = (h - 1) // s + 1, (w - 1) // s + 1
            out.append((stage[0]["conv3"].cout, h, w))
        return out + [(self.image_encoder.out_C, self.vt.H, self.vt.W)]

    def depth_feat(self, rows, shape, depth=None, feat=None):
        return bp.lss_depth_feat_h16(rows, shape, self.vt.D, self.vt.out_channels, depth, feat)

    def image_from_images(self, mats, imgs):
        """Eager image encoder + view transform into the pool image."""
        prepared = self.vt.ranks(mats, 1, self.N)
        depth, feat = self.depth_feat(*self.image_encoder(imgs))
        return self.pool(depth, feat, prepared)

    def forward_images(self, mats, imgs):
        """Eager frame from imgs [N, 3, H, W] fp32 on the device: (boxes, scores, labels, counts) as BEVDet.forward."""
        return self.postprocess(self.dense(self.image_from_images(mats, imgs)))

    def calibrate_heatmap_bias(self, mats, imgs, target_frac=0.014):
        """BEVDet.calibrate_heatmap_bias on the frame of these images."""
        img = self.image_from_images(mats, imgs)
        self.head.calibrate_heatmap_bias(img, self.test_cfg["score_threshold"], target_frac, shape=self.enc_shape)
        return self

    def flops(self):
        """BEVDet.flops (BEV side, its keys unchanged) plus img_backbone (img_stem + img_layers), img_neck, depth_net and
        img_total; frame_total = total + img_total."""
        out = super().flops()
        img = self.image_encoder.flops(self.input_size[0], self.input_size[1], self.N)
        img["img_total"] = img["img_backbone"] + img["img_neck"] + img["depth_net"]
        out.update(img)
        out["frame_total"] = out["total"] + img["img_total"]
        return out


class ImageInput:
    """Mixin of a camera lane (BEVDetHotPath or a subclass) whose depth / feat come from camera images: the lane's
    _depth_feat stage is image encoder -> p3d_lss_depth_feat_h16 on the images in self.imgs [N, 3, H, W] fp32."""

    def _init_images(self):
        H, W = self.model.input_size
        self.imgs = torch.zeros((self.model.N, 3, H, W), dtype=torch.float32, device=self.device)

    def _depth_feat(self):
        m = self.model
        rows, shape = m.image_encoder(self.imgs)
        m.depth_feat(rows, shape, self.depth, self.feat)

    def _put_images(self, imgs):
        """Enqueue the copy of imgs (a device tensor; None: nothing) into the lane's images on its stream."""
        if imgs is not None:
            self.stream.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self.stream):  # after the lane's previous frame, which read the buffer
                self.imgs.copy_(imgs, non_blocking=True)


class FrameInput(ImageInput):
    """ImageInput from decoded camera frames: the lane's _depth_feat stage starts with p3d_image_prep_u8 (the model's
    data_config test pipeline) from the lane's uint8 band buffer self.band into the images.  Only the source rows the
    crop needs (the plan's band) of every camera are copied, as one 2-D copy on the lane's stream before the replay."""

    @classmethod
    def check_plan(cls, model):
        """Raise ValueError when the model has no image prep plan (called before the lane allocates anything)."""
        if getattr(model, "prep_plan", None) is None:
            raise ValueError("%s: the model has no image prep plan (init_weight with a device builds it)" % cls.__name__)

    def _init_band(self):
        plan = self.model.prep_plan
        self.band = torch.zeros((self.model.N, plan.band_rows, plan.src_size[1], 3), dtype=torch.uint8,
                                device=self.device)

    def _depth_feat(self):
        ip.image_prep_u8(self.band, self.model.prep_plan, out=self.imgs)
        super()._depth_feat()

    def check_frames(self, frames):
        """Raise ValueError unless frames is a contiguous uint8 [N, H0, W0, 3] tensor on the lane's device or in pinned
        host memory (a copy from pageable memory would not be asynchronous)."""
        name = type(self).__name__
        plan = self.model.prep_plan
        (H0, W0), N = plan.src_size, self.model.N
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or tuple(frames.shape) != (N, H0, W0, 3) \
                or not frames.is_contiguous():
            raise ValueError("%s: frames must be a contiguous uint8 tensor [%d, %d, %d, 3], got %s %s"
                             % (name, N, H0, W0, getattr(frames, "dtype", type(frames)),
                                tuple(getattr(frames, "shape", ()))))
        if frames.is_cuda:
            if frames.device != self.device:
                raise ValueError("%s: frames on %s, the lane runs on %s" % (name, frames.device, self.device))
        elif not frames.is_pinned():
            raise ValueError("%s: frames in pageable host memory; pass a device tensor or pinned host memory "
                             "(tensor.pin_memory())" % name)

    def _put_frames(self, frames):
        """Enqueue the copy of the band of frames (checked by check_frames) into the lane's band buffer on its stream."""
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):  # after the lane's previous frame, which read the band
            self.copy_band(frames)
            if frames.is_cuda:
                frames.record_stream(self.stream)

    def copy_band(self, frames, out=None):
        """Enqueue the copy of the band rows of frames [N, H0, W0, 3] (checked by check_frames) into out (a band-shaped
        uint8 device tensor; None: the lane's band buffer) on the current stream: one cudaMemcpy2DAsync, a camera per
        row."""
        plan = self.model.prep_plan
        H0, W0 = plan.src_size
        row = W0 * 3
        width = plan.band_rows * row
        dst = self.band if out is None else out
        rc = raw.cudart().cudaMemcpy2DAsync(dst.data_ptr(), width, frames.data_ptr() + plan.band[0] * row, H0 * row,
                                            width, frames.shape[0], 4,  # cudaMemcpyDefault
                                            torch.cuda.current_stream(self.device).cuda_stream)
        if rc != 0:
            raise RuntimeError("cudaMemcpy2DAsync failed (cudaError %d)" % rc)


class BEVDetImageHotPath(ImageInput, BEVDetHotPath):
    """BEVDetHotPath from camera images: one captured CUDA graph from the camera descriptor to the D2H of the boxes, the
    frame being image encoder -> p3d_lss_depth_feat_h16 into the frame's depth / feat -> memset + pool -> encoder -> head
    -> postprocess.  launch(mats, imgs) copies imgs [N, 3, H, W] (a device tensor) into the lane's input buffer on its
    stream first, as CameraFrame.launch copies logits.  Lanes, share_model and accelerate as in BEVDetHotPath."""

    def __init__(self, model, device="cuda", stream=None):
        super().__init__(model, device, stream)
        self._init_images()

    def launch(self, mats, imgs=None):
        """Enqueue one frame: mats = (sensor2ego, cam2imgs, post_rots, post_trans, bda) on the host; imgs: a device tensor
        copied into the frame's input (None: already written there)."""
        self._put_images(imgs)
        self._launch(mats, None, None, "frame")

    def infer(self, mats, imgs=None):
        self.launch(mats, imgs)
        return self.result()


class BEVDetFrameHotPath(FrameInput, BEVDetImageHotPath):
    """BEVDetImageHotPath from decoded camera frames: the captured frame starts with p3d_image_prep_u8 (the model's
    data_config test pipeline: Pillow BICUBIC resize, crop, mmcv.imnormalize, bit-identical to the host's) from the
    lane's uint8 band buffer into the images, then runs BEVDetImageHotPath's frame (FrameInput).  Lanes, share_model and
    accelerate as in BEVDetImageHotPath; the model needs init_weight with a device (its prep plan)."""

    def __init__(self, model, device="cuda", stream=None):
        self.check_plan(model)
        super().__init__(model, device, stream)
        self._init_band()

    def launch_frames(self, sensor2ego, cam2imgs, bda, frames):
        """Enqueue one frame from decoded camera frames [N, H0, W0, 3] uint8 (contiguous; on this device, or in pinned
        host memory, which must stay unchanged until the frame's result is read); the camera matrices as test_mats
        takes them.  Pageable host memory raises ValueError (its copy would not be asynchronous)."""
        self.check_frames(frames)
        mats = self.model.test_mats(sensor2ego, cam2imgs, bda)
        self._put_frames(frames)
        self._launch(mats, None, None, "frame")

    def infer_frames(self, sensor2ego, cam2imgs, bda, frames):
        self.launch_frames(sensor2ego, cam2imgs, bda, frames)
        return self.result()


# ---------------------------------------------------------------------------------------------------------- BEVDet4D
# PARITY UNPINNED, as CONFIG: BEVDet4D (bevdet4d-r50 configs; Paddle3D's bevdet4d.py descends from it) in sequential mode
# with one adjacent frame (multi_adj_frame_id_cfg = (1, 2, 1)): pre_process_net = CustomResNet(numC_input=80,
# num_layer=[2], num_channels=[80], stride=[1]) and the encoder's numC_input = 80 * (num_adj + 1).
CONFIG_4D = dict(CONFIG, backbone=dict(CONFIG["backbone"], in_channels=160),
                 pre_process=dict(num_channels=(80,), strides=(1,), blocks=2), num_adj=1)
CONFIG_4D_BEVDET_NMS = dict(CONFIG_4D, test=TEST_CFG_BEVDET)


class BEVDet4D(BEVDet):
    """Seeded BEVDet4D (CONFIG_4D) in sequential mode (extract_img_feat_sequential): the view transform and pre_process
    give this frame's bev_feat; the previous frame's bev_feat (feat_prev) is shifted into the current ego frame
    (shift_feature: a bilinear grid_sample by the ego motion between the two frames' camera 0) and concatenated after it,
    and the 160-channel concat runs BEVDet's encoder, head and postprocess.  Batch 1.

    Layout on pixel fp16-pair rows: pre_process reads the 96-channel pool image and writes 80 channels into 96-channel
    rows (channels 80..95 of its intermediate images are never written: callers allocate them zero-filled); its last conv
    writes channels [0, 80) of the concat [Y*X, 2*160], the shift channels [80, 160).  bev_feat / feat_prev: the first 96
    channels of the concat's rows ([Y*X, 2*96]; channels 80..95 are not read)."""

    def __init__(self, model_cfg=None, accelerate=False, device="cuda"):
        mc = model_cfg or CONFIG_4D
        if mc.get("num_adj", 1) != 1:
            raise ValueError("BEVDet4D runs one adjacent frame (num_adj = 1), got num_adj = %r" % mc.get("num_adj"))
        super().__init__(mc, accelerate, device)
        pp, b = mc["pre_process"], mc["backbone"]
        X, Y, Z = self.vt.grid
        self.pre_process = BEVDetEncoder(Z * mc["channels"], pp["num_channels"], pp["strides"], pp["blocks"], None,
                                         bn_eps=b["bn_eps"], in_pad=self.pool_C, row_pad=self.pool_C)
        self.bev_C = pp["num_channels"][-1]
        self.hist_C = self.pool_C
        if (any(s != 1 for s in pp["strides"]) or self.bev_C > self.hist_C or self.bev_C % 16
                or self.encoder.in_channels != 2 * self.bev_C or self.encoder.in_pad != 2 * self.bev_C):
            raise ValueError("BEVDet4D: the encoder takes cat([bev_feat, shifted feat_prev]) of %d + %d channels"
                             % (self.bev_C, self.bev_C))

    def init_weight(self, seed=0, bn_gain=1.0, device=None):
        super().init_weight(seed=seed, bn_gain=bn_gain, device=device)
        rng = np.random.default_rng([seed, 4])
        dev = None if device is False else (device or self.device)
        for c in self.pre_process.convs():
            c.init(rng, dev, bn_gain=bn_gain)
        return self

    def export_numpy(self):
        return dict(super().export_numpy(), pre_process=self.pre_process.export_numpy()["backbone"])

    # ---- stages, device in / device out
    def pre_buffers(self):
        """Zero-filled intermediate images of pre_process ([Y*X, 2*96] each; their padding channels stay zero)."""
        _, Y, X, pc = self.image_shape
        z = lambda: torch.zeros((Y * X, 2 * pc), dtype=torch.float16, device=self.device)  # noqa: E731
        bufs = []
        for si, stage in enumerate(self.pre_process.stages):
            bufs.append([])
            for bi, blk in enumerate(stage):
                last = si == len(self.pre_process.stages) - 1 and bi == len(stage) - 1
                d = dict(conv1=z())
                if blk["down"] is not None:
                    d["down"] = z()
                if not last:
                    d["conv2"] = z()
                bufs[-1].append(d)
        return bufs

    def pre(self, image, concat, bufs):
        """pre_process of the pool image into channels [0, 80) of the concat rows."""
        self.pre_process.backbone(image, self.image_shape, bufs, out=(concat, self.encoder.in_pad, 0))

    def shift_desc(self, mats, prev_sensor2keyego=None):
        """pack_shift of this frame: mats as forward takes them (mats[0] = the current sensor2keyego); prev None: the
        start of a sequence (the frame is its own adjacent frame)."""
        lower, interval, _ = self.vt.grid_args()
        prev = mats[0] if prev_sensor2keyego is None else prev_sensor2keyego
        return bp.pack_shift(mats[0], prev, mats[4], lower, interval)

    def shift(self, feat_prev, tf, concat):
        """shift_feature of feat_prev (the history rows, or None: the concat's own bev_feat) into channels [80, 160)."""
        _, Y, X, ec = self.enc_shape
        src, in_c = (concat, ec) if feat_prev is None else (feat_prev, self.hist_C)
        bp.bev_shift_h16(src, (1, Y, X, in_c), tf, self.bev_C, out_h16=concat, out_channels=ec, out_c0=self.bev_C)

    def concat_of(self, image, mats, prev_sensor2keyego, feat_prev=None):
        """Eager: the concat rows [Y*X, 2*160] of a frame from its pool image (feat_prev None: the start of a sequence)."""
        _, Y, X, ec = self.enc_shape
        concat = torch.empty((Y * X, 2 * ec), dtype=torch.float16, device=self.device)
        self.pre(image, concat, self.pre_buffers())
        tf = torch.from_numpy(self.shift_desc(mats, None if feat_prev is None else prev_sensor2keyego)).to(self.device)
        self.shift(feat_prev, tf, concat)
        return concat

    def forward_concat(self, concat):
        """Eager: (boxes, scores, labels, counts) of the concat rows and bev_feat [Y*X, 2*96], their first 96 channels."""
        bev_feat = concat[:, :2 * self.hist_C].contiguous()
        return self.postprocess(self.dense(concat)), bev_feat

    def encoder_input(self, mats, prev_sensor2keyego, logits, tran_feat, feat_prev=None):
        """Eager: the concat rows [Y*X, 2*160] of a frame (feat_prev None: the start of a sequence)."""
        return self.concat_of(self.image(mats, logits, tran_feat), mats, prev_sensor2keyego, feat_prev)

    def forward(self, mats, prev_sensor2keyego, logits, tran_feat, feat_prev=None):
        """Eager frame: ((boxes, scores, labels, counts) as BEVDet.forward, bev_feat [Y*X, 2*96]: the next frame's
        feat_prev).  mats = (sensor2keyego, cam2imgs, post_rots, post_trans, bda) of this frame; prev_sensor2keyego [1, N, 4,
        4]: the previous frame's cameras in this frame's ego (ops.bev_pool_v2.sensor2keyegos); feat_prev None starts a
        sequence (bev_feat is its own adjacent frame and prev_sensor2keyego is not used)."""
        return self.forward_concat(BEVDet4D.encoder_input(self, mats, prev_sensor2keyego, logits, tran_feat, feat_prev))

    def calibrate_heatmap_bias(self, mats, logits, tran_feat, target_frac=0.014):
        """BEVDet.calibrate_heatmap_bias on the start frame of a sequence with these inputs."""
        x = BEVDet4D.encoder_input(self, mats, None, logits, tran_feat)
        self.head.calibrate_heatmap_bias(x, self.test_cfg["score_threshold"], target_frac, shape=self.enc_shape)
        return self

    def flops(self):
        """BEVDet.flops (the encoder's first stage at 160 input channels) plus pre_process (five 3x3 convs 80 -> 80 at the
        pool image's size; the Cin padding 80 -> 96 is not counted)."""
        out = super().flops()
        _, H, W, _ = self.image_shape
        out["pre_process"] = sum(2.0 * H * W * c.cin * c.cout * c.k * c.k for c in self.pre_process.convs())
        out["total"] += out["pre_process"]
        return out


class BEVDet4DHotPath(BEVDetHotPath):
    """One BEVDet4D frame as one captured CUDA graph, BEVDetHotPath's frame with the temporal stages: camera descriptor
    H2D -> ranks -> softmax / permute -> memset + pool -> shift descriptor H2D -> pre_process into the concat -> shift
    (the lane's history -> concat channels [80, 160)) -> a 2-D memcpy of the concat's first 96 channels into the history
    -> encoder -> head -> postprocess -> D2H.  The shift reads the old history before the copy replaces it.  Two frame
    graphs over the same buffers: "continue" shifts the history, "start" (the first frame of a sequence) shifts the
    concat's own bev_feat at the transform of prev = curr.  accelerate: the rank graph, then one of the two; the shift
    descriptor is uploaded in the frame graph, so the ranks are still recomputed only when the cameras change.  Each lane
    owns its history: lanes in flight run independent sequences."""

    def __init__(self, model, device="cuda", stream=None):
        super().__init__(model, device, stream)
        _, Y, X, ec = model.enc_shape
        self.concat = torch.empty((Y * X, 2 * ec), dtype=torch.float16, device=self.device)
        self.history = torch.zeros((Y * X, 2 * model.hist_C), dtype=torch.float16, device=self.device)
        self.pre_bufs = model.pre_buffers()  # zero-filled once, outside the graphs
        self.h_shift = torch.zeros((bp.SHIFT_FLOATS,), dtype=torch.float32).pin_memory()
        self.tf = torch.zeros((bp.SHIFT_FLOATS,), dtype=torch.float32, device=self.device)
        self.started = False

    def _frame(self, start=False):
        m = self.model
        self._depth_feat()
        m.pool(self.depth, self.feat, self.prepared, out=self.image)
        self.tf.copy_(self.h_shift, non_blocking=True)
        m.pre(self.image, self.concat, self.pre_bufs)
        m.shift(None if start else self.history, self.tf, self.concat)
        copy_rows(self.history, self.concat, self.history.stride(0) * self.history.element_size())
        return self._dense(self.concat)

    def _parts(self):
        if self.vt.accelerate:
            return {"ranks": self._ranks, "start": lambda: self._frame(True), "continue": self._frame}
        return {"start": lambda: self._full(True), "continue": self._full}

    def launch(self, mats, prev_sensor2keyego=None, logits=None, tran_feat=None, new_sequence=False):
        """Enqueue one frame of this lane's sequence.  mats = (sensor2keyego, cam2imgs, post_rots, post_trans, bda);
        prev_sensor2keyego [1, N, 4, 4]: the previous frame's cameras in this frame's ego (ops.bev_pool_v2.sensor2keyegos);
        new_sequence: this frame starts a sequence (prev_sensor2keyego is not used).  A lane's first frame must start one."""
        self.check_sequence(new_sequence)
        tf = self.model.shift_desc(mats, None if new_sequence else prev_sensor2keyego)
        self._launch(mats, logits, tran_feat, "start" if new_sequence else "continue",
                     host_inputs=lambda: self.h_shift.copy_(torch.from_numpy(tf.reshape(-1))))
        self.started = True

    def check_sequence(self, new_sequence):
        """Raise ValueError when a frame would continue a sequence this lane never started."""
        if not (new_sequence or self.started):
            raise ValueError("%s: the first frame of a lane must start a sequence (new_sequence=True)" % type(self).__name__)

    def infer(self, mats, prev_sensor2keyego=None, logits=None, tran_feat=None, new_sequence=False):
        self.launch(mats, prev_sensor2keyego, logits, tran_feat, new_sequence)
        return self.result()

    def check_status(self, status_host):
        if int(status_host[0]):
            raise RuntimeError("BEVDet4D: an activation left fp16's range (|x| >= 65504) on the fp16-pair path")


# ------------------------------------------------------------------------------------------ BEVDet4D from images
# PARITY UNPINNED, as the configs it combines: BEVDet4D's BEV half (CONFIG_4D) behind BEVDet-R50's image half (CONFIG_IMG).
CONFIG_4D_IMG = dict(CONFIG_4D, img_backbone=IMG_BACKBONE, img_neck=IMG_NECK, depth_net=DEPTH_NET)
CONFIG_4D_IMG_BEVDET_NMS = dict(CONFIG_4D_IMG, test=TEST_CFG_BEVDET)
BDA_IDENTITY = np.eye(3, dtype=np.float32)[None]  # the test pipeline's bda


class BEVDet4DFromImages(BEVDet4D, BEVDetFromImages):
    """BEVDet4D (CONFIG_4D_IMG) from six normalised camera images: BEVDetFromImages's image encoder and
    p3d_lss_depth_feat_h16 in front of BEVDet4D's view transform, pre_process, shift, encoder, head and postprocess.
    Batch 1.  Checks what both parents check (num_adj 1, input_size a multiple of 32, downsample 16, data_config's crop
    equal to input_size).  Seeded weights equal both parents' for the same seed: the image encoder BEVDetFromImages's, the
    BEV half and pre_process BEVDet4D's.  forward() from the depth net's output is BEVDet4D's; the methods whose
    signatures differ between the parents are defined here."""

    def __init__(self, model_cfg=None, accelerate=False, device="cuda"):
        super().__init__(model_cfg or CONFIG_4D_IMG, accelerate, device)

    def encoder_input(self, mats, prev_sensor2keyego, imgs, feat_prev=None):
        """Eager: the concat rows [Y*X, 2*160] of a frame from imgs [N, 3, H, W] fp32 on the device."""
        return self.concat_of(self.image_from_images(mats, imgs), mats, prev_sensor2keyego, feat_prev)

    def forward_images(self, mats, prev_sensor2keyego, imgs, feat_prev=None):
        """Eager frame from imgs [N, 3, H, W] fp32 on the device: ((boxes, scores, labels, counts), bev_feat) as
        BEVDet4D.forward."""
        return self.forward_concat(self.encoder_input(mats, prev_sensor2keyego, imgs, feat_prev))

    def forward_frames(self, sensor2ego, cam2imgs, bda, frames, prev_sensor2keyego=None, feat_prev=None):
        """Eager frame from decoded camera frames [N, H0, W0, 3] uint8 on the device: forward_images on
        images_from_frames(frames) with test_mats (sensor2ego: this frame's sensor2keyego)."""
        return self.forward_images(self.test_mats(sensor2ego, cam2imgs, bda), prev_sensor2keyego,
                                   self.images_from_frames(frames), feat_prev)

    def calibrate_heatmap_bias(self, mats, imgs, target_frac=0.014):
        """BEVDet.calibrate_heatmap_bias on the start frame of a sequence with these images."""
        x = self.encoder_input(mats, None, imgs)
        self.head.calibrate_heatmap_bias(x, self.test_cfg["score_threshold"], target_frac, shape=self.enc_shape)
        return self

    def flops(self):
        """BEVDet4D.flops plus BEVDetFromImages's image keys; frame_total = total (pre_process included) + img_total."""
        out = super().flops()
        out["frame_total"] = out["total"] + out["img_total"]
        return out


def drive_mats(items, test_mats):
    """The pose bookkeeping of one drive, on the host: items = (frames, sensor2ego [N, 4, 4], ego2global [N, 4, 4],
    cam2imgs [N, 3, 3]) per key frame (frames is not read) -> per item (mats, prev_sensor2keyego, new_sequence), what
    BEVDet4DHotPath.launch takes.  mats = test_mats(sensor2keyego, cam2imgs, bda identity) with the frame's cameras in its
    own key ego (ops.bev_pool_v2.sensor2keyegos; the current frame's camera 0 defines the key ego); prev_sensor2keyego
    the previous frame's cameras in this frame's key ego (None on the first item, which starts the sequence)."""
    prev = None
    for _, s2e, e2g, k in items:
        s2e, e2g = np.asarray(s2e, np.float64)[None], np.asarray(e2g, np.float64)[None]
        curr = bp.sensor2keyegos(s2e, e2g, e2g)
        prev_s2ke = None if prev is None else bp.sensor2keyegos(prev[0], prev[1], e2g)
        yield test_mats(curr, np.asarray(k)[None], BDA_IDENTITY), prev_s2ke, prev is None
        prev = (s2e, e2g)


class BEVDet4DImageHotPath(ImageInput, BEVDet4DHotPath):
    """BEVDet4DHotPath from camera images: both frame graphs ("start", "continue") begin with the image encoder ->
    p3d_lss_depth_feat_h16 into the lane's depth / feat (ImageInput), then run BEVDet4DHotPath's frame unchanged (pool ->
    pre_process -> shift -> history copy -> encoder -> head -> postprocess -> D2H).  Each graph holds its own copy of the
    image encoder's activations (one private pool per graph).  Lanes, history and accelerate as in BEVDet4DHotPath."""

    def __init__(self, model, device="cuda", stream=None):
        super().__init__(model, device, stream)
        self._init_images()

    def launch(self, mats, prev_sensor2keyego=None, imgs=None, new_sequence=False):
        """Enqueue one frame of this lane's sequence: BEVDet4DHotPath.launch with imgs [N, 3, H, W] (a device tensor
        copied into the frame's input; None: already written there) in place of the depth net's output."""
        self.check_sequence(new_sequence)
        self._put_images(imgs)
        BEVDet4DHotPath.launch(self, mats, prev_sensor2keyego, None, None, new_sequence)

    def infer(self, mats, prev_sensor2keyego=None, imgs=None, new_sequence=False):
        self.launch(mats, prev_sensor2keyego, imgs, new_sequence)
        return self.result()


class BEVDet4DFrameHotPath(FrameInput, BEVDet4DImageHotPath):
    """BEVDet4DImageHotPath from decoded camera frames: p3d_image_prep_u8 from the lane's band at the head of both frame
    graphs (FrameInput; frames as BEVDetFrameHotPath takes them).  infer_stream runs one drive from frames and ego poses
    with the band's H2D off the critical path."""

    def __init__(self, model, device="cuda", stream=None):
        self.check_plan(model)
        super().__init__(model, device, stream)
        self._init_band()
        self._upload = None

    def launch_frames(self, sensor2ego, cam2imgs, bda, frames, prev_sensor2keyego=None, new_sequence=False):
        """Enqueue one frame of this lane's sequence from decoded camera frames [N, H0, W0, 3] uint8 (contiguous; on this
        device, or in pinned host memory, which must stay unchanged until the frame's result is read); sensor2ego: this
        frame's sensor2keyego; the rest as BEVDet4DImageHotPath.launch.  Pageable host memory raises ValueError."""
        self.check_sequence(new_sequence)
        self.check_frames(frames)
        mats = self.model.test_mats(sensor2ego, cam2imgs, bda)
        self._put_frames(frames)
        self.launch(mats, prev_sensor2keyego, None, new_sequence)

    def infer_frames(self, sensor2ego, cam2imgs, bda, frames, prev_sensor2keyego=None, new_sequence=False):
        self.launch_frames(sensor2ego, cam2imgs, bda, frames, prev_sensor2keyego, new_sequence)
        return self.result()

    def infer_stream(self, items):
        """One drive: items = (frames [N, H0, W0, 3] uint8 pinned, sensor2ego [N, 4, 4], ego2global [N, 4, 4], cam2imgs
        [N, 3, 3]) per key frame, in order (frames as launch_frames takes them; each must stay unchanged until its result
        is yielded).  The first item starts a sequence; bda is the identity; the matrices come from drive_mats.  Yields
        (boxes, scores, labels) per item, in order, as clones.

        The band of item j + 1 is copied on a copy stream into one of two device staging bands while frame j computes
        (the copy is enqueued before the host waits for frame j), then moved into the lane's band by one D2D copy on the
        lane's stream just before its replay; events order the reuse of each staging band (frame.StagedUpload;
        frame.in_flight's schedule on one lane, its slot being the staging band)."""
        if not self.graphs:
            raise RuntimeError("infer_stream needs a captured lane: call capture() first")
        if self._upload is None:
            self._upload = self._new_upload()
        a, b = itertools.tee(items)
        plans = zip((item[0] for item in a), drive_mats(b, self.model.test_mats))
        steps, held = {}, {}  # item -> its matrices until launched; its frames until its result is read
        for kind, i, plan, _, k in in_flight(plans, 1):
            if kind == "submit":
                held[i], steps[i] = plan
                self._upload.stage(k, functools.partial(self._fill, held[i]), first_use=i < 2)
                if i == 0:
                    self._launch_step(steps.pop(0), k)
            else:
                out = self.slot.read(self.check_status, self.done, clone=True)
                del held[i]
                if i + 1 in steps:
                    self._launch_step(steps.pop(i + 1), k ^ 1)
                yield out

    def _new_upload(self):
        """The staged upload of infer_stream: two staging bands."""
        return StagedUpload([self.band])

    def _fill(self, frames, dev, host):
        """StagedUpload fill of one drive item: check its frames and enqueue the H2D of their band into dev."""
        self.check_frames(frames)
        self.copy_band(frames, out=dev[0])
        if frames.is_cuda:
            frames.record_stream(torch.cuda.current_stream(self.device))

    def _launch_step(self, step, k):
        """Launch the frame whose input is in staging set k: its D2D into the lane's input on the lane's stream, then the
        replay (BEVDet4DImageHotPath.launch).  step = (mats, prev_sensor2keyego, new_sequence)."""
        mats, prev, new_sequence = step
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        self._upload.unstage(k, self.stream)  # after the lane's previous frame, which read the input
        self.launch(mats, prev, None, new_sequence)


# ------------------------------------------------------------------------------------------ from JPEG camera files
class JpegInput(FrameInput):
    """FrameInput from the bytes of N JPEG files (ops/jpeg): the lane's _depth_feat stage clears the lane's JPEG status
    words, decodes the plan's band of every camera from the lane's byte buffer into the band (p3d_jpeg_decode_u8,
    bit-identical to Pillow's decode), copies the status words back with the frame, then runs FrameInput's stage.  The
    compressed bytes and the descriptors go H2D from pinned staging before the replay; one graph serves any compressed
    lengths and tables.  max_bytes: the lane's capacity per camera file.  A corrupt file fails that frame's result()
    with a RuntimeError naming the camera; the lane's next frame is unaffected."""

    DEFAULT_MAX_BYTES = 2 << 20

    def _init_jpeg(self, max_bytes):
        self.jpeg_max_bytes = int(max_bytes)
        if self.jpeg_max_bytes < 1:
            raise ValueError("%s: max_bytes %d" % (type(self).__name__, self.jpeg_max_bytes))
        N = self.model.N
        dev = self.device
        self.jpeg_data = torch.zeros((N * self.jpeg_max_bytes,), dtype=torch.uint8, device=dev)
        self.jpeg_desc = torch.zeros((N * jpeg.DESC_DTYPE.itemsize,), dtype=torch.uint8, device=dev)
        self.jpeg_status = torch.zeros((N,), dtype=torch.int32, device=dev)
        self.h_jpeg_data = torch.empty((N * self.jpeg_max_bytes,), dtype=torch.uint8).pin_memory()
        self.h_jpeg_desc = torch.empty((N * jpeg.DESC_DTYPE.itemsize,), dtype=torch.uint8).pin_memory()
        self.h_jpeg_status = torch.zeros((N,), dtype=torch.int32).pin_memory()
        self._jpeg_copied = None  # event after the last H2D from the pinned staging

    def _depth_feat(self):
        plan = self.model.prep_plan
        self.jpeg_status.zero_()
        jpeg.jpeg_decode_u8(self.jpeg_data, self.jpeg_desc, self.model.N, plan.src_size, rows=plan.band, out=self.band,
                            status=self.jpeg_status, max_bytes=self.jpeg_max_bytes)
        self.h_jpeg_status.copy_(self.jpeg_status, non_blocking=True)
        super()._depth_feat()

    def check_status(self, status_host):
        bad = [(i, int(s)) for i, s in enumerate(self.h_jpeg_status.tolist()) if s]
        if bad:
            raise RuntimeError("%s: JPEG decode failed: %s" % (type(self).__name__, "; ".join(
                "camera %d: corrupt data (status 0x%x: %s)" % (i, s, jpeg.status_reason(s)) for i, s in bad)))
        super().check_status(status_host)

    def pack_jpegs(self, jpegs, data=None, desc=None):
        """Parse N JPEG files (bytes or uint8 numpy arrays) and write their bytes and descriptors into the pinned
        buffers data / desc (default: the lane's, once its previous H2D has read them).  Returns the bytes used.  ValueError (nothing enqueued) for a rejected
        header, a size other than the plan's src_size, a wrong count or a file longer than max_bytes."""
        name = type(self).__name__
        N = self.model.N
        if len(jpegs) != N:
            raise ValueError("%s: %d JPEG files, want %d" % (name, len(jpegs), N))
        blobs = [f if isinstance(f, bytes) else (f.tobytes() if isinstance(f, np.ndarray) else bytes(f)) for f in jpegs]
        for i, b in enumerate(blobs):
            if len(b) > self.jpeg_max_bytes:
                raise ValueError("%s: camera %d: %d bytes exceed the lane's capacity of %d per file"
                                 % (name, i, len(b), self.jpeg_max_bytes))
        if data is None:
            data, desc = self.h_jpeg_data, self.h_jpeg_desc
            if self._jpeg_copied is not None:
                self._jpeg_copied.synchronize()  # the previous H2D from the lane's staging has read it
        try:
            raw_data, d, _ = jpeg.batch(blobs, self.model.prep_plan.src_size, out=data.numpy())
        except ValueError as e:
            raise ValueError("%s: %s" % (name, e)) from None
        desc.numpy()[:] = d.view(np.uint8)
        return len(raw_data)

    def _put_jpegs(self, nbytes):
        """Enqueue the H2D of the packed bytes and descriptors into the lane's buffers on its stream."""
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):  # after the lane's previous frame, which read the buffers
            self.jpeg_data[:nbytes].copy_(self.h_jpeg_data[:nbytes], non_blocking=True)
            self.jpeg_desc.copy_(self.h_jpeg_desc, non_blocking=True)
            self._jpeg_copied = torch.cuda.Event()
            self._jpeg_copied.record(self.stream)


class BEVDetJpegHotPath(JpegInput, BEVDetFrameHotPath):
    """BEVDetFrameHotPath from the bytes of six JPEG camera files: the captured frame starts with the device JPEG decode
    of the prep plan's band into the lane's band (JpegInput), then runs BEVDetFrameHotPath's frame.  Lanes, share_model
    and accelerate as in BEVDetFrameHotPath."""

    def __init__(self, model, device="cuda", stream=None, max_bytes=JpegInput.DEFAULT_MAX_BYTES):
        super().__init__(model, device, stream)
        self._init_jpeg(max_bytes)

    def launch_jpegs(self, sensor2ego, cam2imgs, bda, jpegs):
        """Enqueue one frame from N JPEG files (bytes or uint8 numpy arrays, in camera order); the camera matrices as
        test_mats takes them.  The files are parsed and copied to pinned staging here (ValueError before anything is
        enqueued when one is rejected or too long)."""
        nbytes = self.pack_jpegs(jpegs)
        mats = self.model.test_mats(sensor2ego, cam2imgs, bda)
        self._put_jpegs(nbytes)
        self._launch(mats, None, None, "frame")

    def infer_jpegs(self, sensor2ego, cam2imgs, bda, jpegs):
        self.launch_jpegs(sensor2ego, cam2imgs, bda, jpegs)
        return self.result()


class BEVDet4DJpegHotPath(JpegInput, BEVDet4DFrameHotPath):
    """BEVDet4DFrameHotPath from the bytes of six JPEG camera files (JpegInput at the head of both frame graphs).
    infer_stream runs one drive from JPEG files and ego poses with the H2D of the next item's bytes on a copy stream
    while the current frame computes: its items carry N JPEG files (as launch_jpegs takes them) in place of the frames."""

    def __init__(self, model, device="cuda", stream=None, max_bytes=JpegInput.DEFAULT_MAX_BYTES):
        super().__init__(model, device, stream)
        self._init_jpeg(max_bytes)

    def launch_jpegs(self, sensor2ego, cam2imgs, bda, jpegs, prev_sensor2keyego=None, new_sequence=False):
        """Enqueue one frame of this lane's sequence from N JPEG files; the rest as BEVDet4DFrameHotPath.launch_frames."""
        self.check_sequence(new_sequence)
        nbytes = self.pack_jpegs(jpegs)
        mats = self.model.test_mats(sensor2ego, cam2imgs, bda)
        self._put_jpegs(nbytes)
        self.launch(mats, prev_sensor2keyego, None, new_sequence)

    def infer_jpegs(self, sensor2ego, cam2imgs, bda, jpegs, prev_sensor2keyego=None, new_sequence=False):
        self.launch_jpegs(sensor2ego, cam2imgs, bda, jpegs, prev_sensor2keyego, new_sequence)
        return self.result()

    def _new_upload(self):
        """The staged upload of infer_stream: the files' bytes and descriptors through pinned and device staging."""
        return StagedUpload([self.jpeg_data, self.jpeg_desc], pinned=True)

    def _fill(self, jpegs, dev, host):
        """StagedUpload fill of one drive item: parse its files into the pinned buffers host, then enqueue the H2D of the
        bytes used and of the descriptors into dev."""
        n = self.pack_jpegs(jpegs, *host)
        dev[0][:n].copy_(host[0][:n], non_blocking=True)
        dev[1].copy_(host[1], non_blocking=True)
        return n, len(host[1])
