"""BEVDet inference on one GPU from the depth net's output on (BEVDet-R50's BEV half, PARITY UNPINNED: the model values in
CONFIG are recalled from BEVDet's bevdet-r50 config, which Paddle3D's configs/bevdet descend from; they were not checked
against either file):

    camera descriptor H2D -> p3d_lss_prepare -> depth softmax / permute -> bev_pool straight into the pixel fp16-pair image
    [128 x 128 x 96] (channels 80..95 zero) -> CustomResNet (BasicBlocks, residual added in the conv epilogue) -> FPN_LSS
    (bilinear x4 / x2 with align_corners on the pair rows) -> CenterHead (dense_head.DenseRPNHead with this encoder as its
    trunk) -> centerpoint_postprocess_device -> boxes

BEVDetHotPath captures all of it, from the descriptor upload to the D2H copy of the boxes, as one CUDA graph.  The
postprocess is the custom op Paddle3D's predict_by_custom_op calls (rotated NMS per task), not BEVDet's scale-NMS."""
import numpy as np
import torch

from . import synth
from .dense_head import COMMON_HEADS, DenseRPNHead, _Conv
from .lss import LSSViewTransformer
from .ops import bev_pool_v2 as bp
from .ops import centerpoint_postprocess as cpp
from .ops import dense_conv as dc
from .ops import sparse_nn as sp
from .pipeline import _count_graph_nodes

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


def round32(c):
    return (int(c) + 31) // 32 * 32


class BEVDetEncoder:
    """CustomResNet (BasicBlocks: relu(bn2(conv2(relu(bn1(conv1(x))))) + identity); the first block of a stage has a 3x3
    stride-s conv1 and a 3x3 stride-s Conv2d with bias as its identity branch) + FPN_LSS (cat([x0, up4(x2)]), two 3x3
    ConvModules, up2, a 3x3 ConvModule and a 1x1 conv with bias), on pixel fp16-pair rows.  A DenseRPNHead trunk.
    in_pad: channels of the input image rows (the pool image's, in_channels rounded up to 32); the first stage's weights
    are zero-padded on Cin to it once, when they are packed."""

    def __init__(self, in_channels, num_channels, strides, blocks, fpn_out, scale_factor, input_feature_index,
                 extra_upsample, bn_eps=1e-5, in_pad=None):
        self.in_channels, self.in_pad = in_channels, in_pad or round32(in_channels)
        self.scale_factor, self.extra_upsample = scale_factor, extra_upsample
        self.index = tuple(input_feature_index)
        self.stages = []
        cin = in_channels
        for si, (cout, s) in enumerate(zip(num_channels, strides)):
            pad = self.in_pad if si == 0 else None
            stage = [dict(conv1=_Conv(cin, cout, 3, s, 1, bn_eps=bn_eps, cin_pad=pad),
                          conv2=_Conv(cout, cout, 3, 1, 1, bn_eps=bn_eps),  # ReLU after the residual
                          down=_Conv(cin, cout, 3, s, 1, bias=True, relu=False, cin_pad=pad))]
            for _ in range(blocks - 1):
                stage.append(dict(conv1=_Conv(cout, cout, 3, 1, 1, bn_eps=bn_eps), conv2=_Conv(cout, cout, 3, 1, 1, bn_eps=bn_eps),
                                  down=None))
            self.stages.append(stage)
            cin = cout
        self.stage_channels = tuple(num_channels)
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

    @staticmethod
    def _block(blk, x, shape):
        b = shape[0]
        t, _, (_, oh, ow) = blk["conv1"](x, shape)
        cout = blk["conv1"].cout
        idn = x if blk["down"] is None else blk["down"](x, shape)[0]
        y, _, _ = blk["conv2"](t, (b, oh, ow, cout), residual=idn, res_channels=cout)
        return y, (b, oh, ow, cout)

    def backbone(self, x, shape):
        """CustomResNet: the pixel image of every stage's output, [(rows, (B, H, W, C))]."""
        feats = []
        for stage in self.stages:
            for blk in stage:
                x, shape = self._block(blk, x, shape)
            feats.append((x, shape))
        return feats

    def __call__(self, x, shape, first=None):
        """x: pixel fp16-pair rows [B*H*W, 2*in_pad], shape = (B, H, W, in_pad).  Returns (FPN_LSS output rows, shape)."""
        if first is not None or int(shape[3]) != self.in_pad:
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
        self.encoder = BEVDetEncoder(Z * mc["channels"], b["num_channels"], b["strides"], b["blocks"], f["out_channels"],
                                     f["scale_factor"], f["input_feature_index"], f["extra_upsample"], b["bn_eps"], self.pool_C)
        if self.encoder.cat_channels != f["in_channels"]:
            raise ValueError("FPN_LSS in_channels %d, the concat has %d" % (f["in_channels"], self.encoder.cat_channels))
        self.head = DenseRPNHead(in_channels=f["out_channels"], tasks=h["tasks"], share_conv_channel=h["share_conv_channel"],
                                 bev_depth=1, trunk=self.encoder)
        self.test_cfg = dict(mc["test"])
        self.label_off = synth.label_offsets(list(h["tasks"]))
        self.image_shape = (1, Y, X, self.pool_C)

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
        return self.encoder(image, self.image_shape)

    def dense(self, image):
        """Pool image -> dict name -> per-task [1, k, 128, 128] fp32 head planes."""
        return self.head.forward_h16(image, self.image_shape)

    def postprocess(self, h):
        tc = self.test_cfg
        return cpp.centerpoint_postprocess_device(
            h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], tc["voxel_size"], tc["point_cloud_range"],
            tc["post_center_limit_range"], self.label_off, tc["down_ratio"], tc["score_threshold"],
            tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"], True)

    def forward(self, mats, logits, tran_feat):
        """Eager frame: (boxes, scores, labels, counts) on the device, worst-case sized (counts[-1] rows valid)."""
        return self.postprocess(self.dense(self.image(mats, logits, tran_feat)))

    def calibrate_heatmap_bias(self, mats, logits, tran_feat, target_frac=0.014):
        """DenseRPNHead.calibrate_heatmap_bias on this frame: ~1.4 % of the cells above the score threshold, as the LiDAR
        frames do.  Weights stay seeded and are exported unchanged to the CPU arm."""
        img = self.image(mats, logits, tran_feat)
        self.head.calibrate_heatmap_bias(img, self.test_cfg["score_threshold"], target_frac, shape=self.image_shape)
        return self

    def flops(self):
        """Algorithmic flops (2 x MACs) of the dense part: backbone (CustomResNet with its identity convs), FPN_LSS and
        the head (shared conv, the 36 ConvModules, the output convs).  The Cin padding 80 -> 96 is not counted."""
        out = dict(backbone=0.0, fpn=0.0, head_shared=0.0, head_convmodules=0.0, head_output=0.0)
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
        px = h1 * h1
        sh = self.head.shared
        out["head_shared"] = 2.0 * px * sh.cin * sh.cout * sh.k * sh.k
        for hs in self.head.heads:
            for _, a, f in hs:
                out["head_convmodules"] += 2.0 * px * a.cin * a.cout * a.k * a.k
                out["head_output"] += 2.0 * px * f.cin * f.cout * f.k * f.k
        out["head"] = out["head_shared"] + out["head_convmodules"] + out["head_output"]
        out["total"] = out["backbone"] + out["fpn"] + out["head"]
        return out

    def head_planes(self):
        return sum(sum(c for _, c in COMMON_HEADS) + n for n in self.head.tasks)


class BEVDetHotPath:
    """One BEVDet frame as one captured CUDA graph on its own stream: camera descriptor H2D -> p3d_lss_prepare -> depth
    softmax / permute -> memset + pool into the pixel image -> encoder -> head -> postprocess -> one D2H of boxes [6 x 83,
    9], scores, labels, counts and the status word.  Any calibration replays the same graph.  accelerate (the model's
    view transformer built with accelerate=True): two graphs, ranks (replayed only when the camera matrices differ from
    the last ones) and the rest.  Several lanes may share one model (share_model), each with its own buffers and stream.
    The status word is the device's fp16-pair overflow flag (ops.sparse_nn.status_tensor), which stays set once raised."""

    def __init__(self, model, device="cuda", stream=None):
        self.model = model
        self.device = torch.device(device)
        self.stream = stream or torch.cuda.Stream(self.device)
        vt, N = model.vt, model.N
        nd = N * bp.CAM_FLOATS + 9
        self.h_desc = torch.zeros((nd,), dtype=torch.float32).pin_memory()
        self.desc = torch.zeros((nd,), dtype=torch.float32, device=self.device)
        D, H, W, C = vt.D, vt.H, vt.W, vt.out_channels
        self.logits = torch.zeros((N, D, H, W), dtype=torch.float32, device=self.device)
        self.tran_feat = torch.zeros((N, C, H, W), dtype=torch.float32, device=self.device)
        self.depth = torch.empty_like(self.logits)
        self.feat = torch.empty((N, H, W, C), dtype=torch.float32, device=self.device)
        _, Y, X, pc = model.image_shape
        self.image = torch.empty((Y * X, 2 * pc), dtype=torch.float16, device=self.device)
        rows = len(model.label_off) * model.test_cfg["nms_post_max_size"]
        self.h_boxes = torch.zeros((rows, 9), dtype=torch.float32).pin_memory()
        self.h_scores = torch.zeros((rows,), dtype=torch.float32).pin_memory()
        self.h_labels = torch.zeros((rows,), dtype=torch.int64).pin_memory()
        self.h_counts = torch.zeros((len(model.label_off) + 1,), dtype=torch.int32).pin_memory()
        self.h_status = torch.zeros((1,), dtype=torch.int32).pin_memory()
        self.graphs, self.graph_nodes, self.prepared, self.last, self.out = {}, None, None, None, None
        self.done = torch.cuda.Event()

    def share_model(self, other):
        self.model = other.model
        return self

    # ---- stages, as they are captured
    def _ranks(self):
        self.desc.copy_(self.h_desc, non_blocking=True)
        self.prepared = self.model.vt._prepare(self.desc, 1, self.model.N)

    def _frame(self):
        m = self.model
        bp.lss_depth_feat(self.logits, self.tran_feat, self.depth, self.feat)
        m.pool(self.depth, self.feat, self.prepared, out=self.image)
        h = m.dense(self.image)
        boxes, scores, labels, counts = m.postprocess(h)
        self.out = dict(boxes=boxes, scores=scores, labels=labels, counts=counts, head=h)
        self.h_boxes.copy_(boxes, non_blocking=True)
        self.h_scores.copy_(scores, non_blocking=True)
        self.h_labels.copy_(labels, non_blocking=True)
        self.h_counts.copy_(counts, non_blocking=True)
        self.h_status.copy_(sp.status_tensor(self.device), non_blocking=True)

    def _full(self):
        self._ranks()
        self._frame()

    def capture(self, count_nodes=False):
        """Warm up eagerly (sizes the workspaces), then capture the frame graph (accelerate: the rank graph and the rest).
        count_nodes: node counts by type of the graphs in self.graph_nodes."""
        parts = {"ranks": self._ranks, "frame": self._frame} if self.model.vt.accelerate else {"frame": self._full}
        with torch.cuda.stream(self.stream):
            self._full()
            self.stream.synchronize()
            for name, fn in parts.items():
                g = torch.cuda.CUDAGraph(keep_graph=True) if count_nodes else torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=self.stream):
                    fn()
                self.graphs[name] = g
                if count_nodes:
                    nodes = _count_graph_nodes(g.raw_cuda_graph())
                    self.graph_nodes = nodes if self.graph_nodes is None else {k: self.graph_nodes[k] + nodes[k] for k in nodes}
        self.stream.synchronize()
        self.last = None
        return self

    def launch(self, mats, logits=None, tran_feat=None):
        """Enqueue one frame on self.stream.  mats = (sensor2ego, cam2imgs, post_rots, post_trans, bda) of one sample on
        the host; logits [N, D, H, W] / tran_feat [N, C, H, W]: device tensors copied into the frame's inputs (None:
        already written there)."""
        packed = bp.pack_cameras(*mats)
        self.done.synchronize()  # the previous frame's H2D has read h_desc and its D2H has landed
        self.stream.wait_stream(torch.cuda.current_stream(self.device))  # inputs written on the caller's stream
        with torch.cuda.stream(self.stream):
            if logits is not None:
                self.logits.copy_(logits, non_blocking=True)
            if tran_feat is not None:
                self.tran_feat.copy_(tran_feat, non_blocking=True)
            if not self.model.vt.accelerate:
                self.h_desc.copy_(torch.from_numpy(packed))
                self.graphs["frame"].replay()
            else:
                if self.last is None or not np.array_equal(self.last, packed):
                    self.h_desc.copy_(torch.from_numpy(packed))
                    self.graphs["ranks"].replay()
                    self.last = packed
                self.graphs["frame"].replay()
            self.done.record(self.stream)

    def result(self):
        """Wait for the last launched frame: (boxes [K, 9], scores [K], labels [K]) host tensors owned by the lane (valid
        until its next launch); raises from check_status."""
        self.done.synchronize()
        self.check_status(self.h_status)
        k = int(self.h_counts[-1])
        return self.h_boxes[:k], self.h_scores[:k], self.h_labels[:k]

    def infer(self, mats, logits=None, tran_feat=None):
        self.launch(mats, logits, tran_feat)
        return self.result()

    def check_status(self, status_host):
        """Raise when an activation left fp16's range on the fp16-pair path (never a silent wrong result)."""
        if int(status_host[0]):
            raise RuntimeError("BEVDet: an activation left fp16's range (|x| >= 65504) on the fp16-pair path")
