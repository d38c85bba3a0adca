"""SURVEY.md §8f-1: the dense part of CenterPoint between the BEV tensor and the postprocess —
SecondBackbone (backbones/second_backbone.py:72-120), SecondFPN (necks/second_fpn.py:99-160, use_conv_for_no_stride)
and CenterHead (detection/centerpoint/center_head.py:43-220) — as a chain of `ops.dense_conv.dense_conv2d` launches
with BatchNorm folded into the conv epilogue.  Same constructor vocabulary as the reference's yml
(configs/centerpoint/centerpoint_voxels_0075voxel_nuscenes_10sweep.yml:127-162).  Default arithmetic: fp16 (hi, lo')
pair operands on wgmma (csrc/dense_conv_f16.cu, `f16=True`); the tf32-pair kernels stay selectable
(`f16=False`) for data outside fp16's range.  The 36 ConvModules of the heads run as ONE 64 -> 2304 convolution and
the 36 output convs as one launch (forward: tap-as-N tensor-core kernel on the fp16-pair path, CUDA cores on the tf32
one); forward_per_head keeps the layer-by-layer form for the parity tests."""
import numpy as np
import torch

from .ops import dense_conv as dc

COMMON_HEADS = (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))  # yml:157-162, then hm per task


class _Conv:
    """Conv2D / Conv2DTranspose (+ BatchNorm2D eval) (+ ReLU) with seeded parameters."""

    def __init__(self, cin, cout, k, stride=1, padding=0, bias=False, bn_eps=None, relu=True, up=1, f16=True, transposed=False,
                 cin_pad=None, cout_pad=None):
        """transposed: a stride-1 Conv2DTranspose (weight [Cin, Cout, k, k]); with k = 1 it runs as a 1x1 conv whose packed
        weight is the transpose (up > 1 implies a transposed conv).  cin_pad: the packed weight is zero-padded on Cin to
        this many channels (an input image whose rows carry zero padding channels); the exported weight keeps cin.
        cout_pad: the device conv computes this many output channels, the ones past cout with zero weights, bias and
        shift (an fp16-pair output needs Cout % 16 == 0); the exported parameters keep cout."""
        self.cin, self.cout, self.k, self.stride, self.padding, self.up = cin, cout, k, stride, padding, up
        self.cin_pad, self.cout_pad = cin_pad, cout_pad
        self.transposed = transposed or up > 1
        self.has_bias, self.bn_eps, self.relu = bias, bn_eps, relu
        self.f16 = f16 and cout >= 16  # the 1-3 channel output convs of the heads run on the CUDA cores (forward)
        self.n_tile = dc.n_tile_for_f16(cout) if self.f16 else dc.n_tile_for(cout)
        self.np = None
        self.dev = None

    def init(self, rng, device=None, randomize_bn=False, bias_value=None, bn_gain=1.0):
        """Seeded parameters (numpy); with a device also the packed tensor-core image and the folded epilogue."""
        cin, cout, k = self.cin, self.cout, self.k
        bound = 1.0 / np.sqrt(cin * k * k)  # build_conv_layer "uniform" (second_backbone.py:43-48)
        w = rng.uniform(-bound, bound, size=self.weight_shape()).astype(np.float32)
        b = None
        if self.has_bias:
            b = (np.full(cout, bias_value, np.float32) if bias_value is not None
                 else rng.uniform(-bound, bound, size=cout).astype(np.float32))
        bn = None
        if self.bn_eps is not None:
            if randomize_bn:
                g, bt = rng.uniform(0.5, 1.5, cout), rng.uniform(-0.2, 0.2, cout)
                m, v = rng.uniform(-0.1, 0.1, cout), rng.uniform(0.5, 1.5, cout)
            else:
                g, bt, m, v = np.ones(cout), np.zeros(cout), np.zeros(cout), np.ones(cout)
            g = g * bn_gain
            bn = dict(gamma=g.astype(np.float32), beta=bt.astype(np.float32), mean=m.astype(np.float32),
                      var=v.astype(np.float32))
        return self.set_parameters(w, b, bn, device)

    def weight_shape(self):
        """Paddle's weight layout: [Cin, Cout, k, k] for a Conv2DTranspose, [Cout, Cin, k, k] for a Conv2D."""
        return (self.cin, self.cout, self.k, self.k) if self.transposed else (self.cout, self.cin, self.k, self.k)

    def set_parameters(self, w, b=None, bn=None, device=None):
        """Parameters in Paddle's layouts, float32 numpy: weight (weight_shape()), bias [Cout] (with bias), bn dict gamma /
        beta / mean / var [Cout] (with BatchNorm).  They become self.np and, with a device, the packed tensor-core image
        and the folded epilogue (self.dev); without one self.dev is left as it is."""
        cout, shape = self.cout, self.weight_shape()
        p = dict(weight=w, bias=b, stride=self.stride, padding=self.padding, up=self.up, relu=self.relu, bn=None,
                 transposed=self.transposed)
        if self.bn_eps is not None:
            p["bn"] = dict(bn, eps=self.bn_eps)
        self.np = p
        if device is None:
            return self
        # fold: y = conv * s + ((bias - mean) * s + beta), s = gamma / sqrt(var + eps)   (fp64 on the host)
        s = np.ones(cout)
        t = np.zeros(cout) if b is None else b.astype(np.float64)
        if p["bn"] is not None:
            bn = p["bn"]
            s = bn["gamma"].astype(np.float64) / np.sqrt(bn["var"].astype(np.float64) + bn["eps"])
            t = (t - bn["mean"]) * s + bn["beta"]
        if self.f16:
            pack = dc.pack_deconv_weight_f16 if self.transposed else dc.pack_conv_weight_f16
        else:
            pack = dc.pack_deconv_weight if self.transposed else dc.pack_conv_weight
        wd = w
        if self.cin_pad and self.cin_pad > self.cin:
            ax = 0 if self.transposed else 1
            wd = np.zeros(shape[:ax] + (self.cin_pad,) + shape[ax + 1:], np.float32)
            wd[(slice(None),) * ax + (slice(0, self.cin),)] = w
        if self.cout_pad and self.cout_pad > cout:
            if self.transposed:
                raise ValueError("cout_pad: Conv2D weights only")
            wp = np.zeros((self.cout_pad,) + wd.shape[1:], np.float32)
            wp[:cout] = wd
            wd = wp
            s, t = np.concatenate([s, np.ones(self.cout_pad - cout)]), np.concatenate([t, np.zeros(self.cout_pad - cout)])
        self.dev = dict(
            packed=pack(torch.from_numpy(wd).to(device), self.n_tile),
            scale=torch.from_numpy(s.astype(np.float32)).to(device) if p["bn"] is not None else None,
            shift=torch.from_numpy(t.astype(np.float32)).to(device) if (p["bn"] is not None or b is not None) else None)
        return self

    def __call__(self, x_split, shape, **kw):
        d = self.dev
        if self.f16:
            if "out_split" in kw:
                kw["out_h16"] = kw.pop("out_split")
            return dc.dense_conv2d_f16(x_split, shape, d["packed"], self.cout_pad or self.cout, self.n_tile, self.k, self.stride,
                                       self.padding, self.up, d["scale"], d["shift"], self.relu, **kw)
        return dc.dense_conv2d(x_split, shape, d["packed"], self.cout, self.n_tile, self.k, self.stride, self.padding, self.up,
                               d["scale"], d["shift"], self.relu, **kw)


class SecondTrunk:
    """SecondBackbone (second_backbone.py:72-120) + SecondFPN (second_fpn.py:99-160): strided 3x3 conv blocks, then one
    deblock per block, all written into one channel-concat pixel image (`out_c0`).  BatchNorm eps 1e-3 throughout."""

    def __init__(self, in_channels, out_channels, layer_nums, downsample_strides, fpn_out_channels, upsample_strides,
                 use_conv_for_no_stride=True, f16=True):
        self.f16 = f16

        def conv(*a, **k):
            return _Conv(*a, f16=f16, **k)
        bn3 = 1e-3
        self.blocks = []
        cin = in_channels
        for cout, n, s in zip(out_channels, layer_nums, downsample_strides):
            blk = [conv(cin, cout, 3, s, 1, bn_eps=bn3)] + [conv(cout, cout, 3, 1, 1, bn_eps=bn3) for _ in range(n)]
            self.blocks.append(blk)
            cin = cout
        self.deblocks = []
        for ci, co, u in zip(out_channels, fpn_out_channels, upsample_strides):
            # stride > 1 -> Conv2DTranspose k = s; stride 1 -> Conv2D k = 1 with use_conv_for_no_stride, else
            # Conv2DTranspose k = 1; stride < 1 -> Conv2D k = stride = round(1 / s) (second_fpn.py:118-139)
            if u > 1:
                self.deblocks.append(conv(ci, co, u, u, 0, bn_eps=bn3, up=u))
            elif u < 1:
                k = int(round(1 / u))
                self.deblocks.append(conv(ci, co, k, k, 0, bn_eps=bn3))
            else:
                self.deblocks.append(conv(ci, co, 1, 1, 0, bn_eps=bn3, transposed=not use_conv_for_no_stride))
        self.fpn_channels = int(sum(fpn_out_channels))

    def convs(self):
        return [c for blk in self.blocks for c in blk] + list(self.deblocks)

    def export_numpy(self):
        return dict(blocks=[[c.np for c in blk] for blk in self.blocks], deblocks=[c.np for c in self.deblocks])

    def __call__(self, x, shape, first=None, out=None, out_channels=None, out_c0=0):
        """x: pixel rows [B*H*W, 2*C] (fp16 pairs or tf32 split) with shape = (B, H, W, C); first replaces the first conv.
        Returns (concat image [B*oH*oW, 2*fpn_channels], (B, oH, oW, fpn_channels)).  out: an existing image of
        out_channels channels per row; the concat is written into its channels [out_c0, out_c0 + fpn_channels) and
        (out, (B, oH, oW, out_channels)) returned."""
        b = shape[0]
        feats = []
        for bi, blk in enumerate(self.blocks):
            for ci, conv in enumerate(blk):
                if bi == 0 and ci == 0 and first is not None:
                    conv = first
                x, _, (b_, oh, ow) = conv(x, shape)
                shape = (b_, oh, ow, conv.cout)
            feats.append((x, shape))
        out_hws = {self.deblock_out_hw(de, fshape[1], fshape[2]) for (_, fshape), de in zip(feats, self.deblocks)}
        if len(out_hws) != 1:
            raise ValueError("the FPN deblocks give feature maps of different sizes %s; the concat needs one size"
                             % sorted(out_hws))
        out_hw = out_hws.pop()
        oc = self.fpn_channels if out is None else int(out_channels)
        cat = out if out is not None else torch.empty((b * out_hw[0] * out_hw[1], 2 * oc),
                                                      dtype=torch.float16 if self.f16 else torch.float32, device=x.device)
        c0 = 0 if out is None else int(out_c0)
        for (f, fshape), de in zip(feats, self.deblocks):
            de(f, fshape, out_split=cat, out_channels=oc, out_c0=c0)
            c0 += de.cout
        return cat, (b, out_hw[0], out_hw[1], oc)

    @staticmethod
    def deblock_out_hw(de, h, w):
        """Output (H, W) of a deblock on an h x w feature map: x up for a transposed conv, the conv geometry otherwise."""
        if de.up > 1:
            return h * de.up, w * de.up
        return (h + 2 * de.padding - de.k) // de.stride + 1, (w + 2 * de.padding - de.k) // de.stride + 1


class DenseRPNHead:
    def __init__(self, in_channels=256, out_channels=(128, 256), layer_nums=(5, 5), downsample_strides=(1, 2),
                 fpn_out_channels=(256, 256), upsample_strides=(1, 2), tasks=(1, 2, 2, 1, 2, 2), share_conv_channel=64,
                 f16=True, with_velocity=None, bev_depth=2, trunk=None, common_heads=COMMON_HEADS):
        """trunk: the network between the BEV image and the shared conv (None: SecondBackbone + SecondFPN from the
        arguments above); another object with SecondTrunk's __call__(x, shape, first=None) / fpn_channels / convs() /
        export_numpy() contract, on pixel fp16-pair rows with bev_depth 1 (bevdet.BEVDetEncoder).  common_heads: the
        CenterHead's (name, channels) heads of every task before its "hm" (CenterHead common_heads); with_velocity
        (default: whether "vel" is among them) decides whether the box decode reads a velocity head."""
        if trunk is not None and (not f16 or bev_depth > 1):
            raise ValueError("a custom trunk runs on the fp16-pair path with bev_depth 1")
        self.tasks = list(tasks)
        self.in_channels, self.bev_depth = in_channels, bev_depth
        self.num_classes = list(tasks)        # CenterHead.num_classes (center_head.py:64)
        self.common_heads = tuple((str(n), int(c)) for n, c in common_heads)
        has_vel = any(n == "vel" for n, _ in self.common_heads)
        if with_velocity is None:
            with_velocity = has_vel
        if with_velocity and not has_vel:
            raise ValueError("with_velocity needs a 'vel' head in common_heads")
        self.with_velocity = bool(with_velocity)  # 'vel' in common_heads (center_head.py:77)
        self.f16 = f16
        if f16 and (share_conv_channel % 32 or not 32 <= share_conv_channel <= 320):
            raise ValueError("the fp16-pair head output convs need share_conv_channel a multiple of 32 and at most 320 "
                             "(got %d); use f16=False" % share_conv_channel)

        def conv(*a, **k):
            return _Conv(*a, f16=f16, **k)
        bn5 = 1e-5
        if trunk is None:
            trunk = SecondTrunk(in_channels, out_channels, layer_nums, downsample_strides, fpn_out_channels,
                                upsample_strides, use_conv_for_no_stride=True, f16=f16)
            self.blocks, self.deblocks = trunk.blocks, trunk.deblocks
        else:
            self.blocks = self.deblocks = None
        self.trunk, self.fpn_channels = trunk, trunk.fpn_channels
        self.shared = conv(self.fpn_channels, share_conv_channel, 3, 1, 1, bias=True, bn_eps=bn5)
        self.heads = []  # per task: list of (name, ConvModule 64->64, final conv 64->classes)
        for ncls in self.tasks:
            hs = []
            for name, c in list(self.common_heads) + [("hm", ncls)]:
                hs.append((name, conv(share_conv_channel, share_conv_channel, 3, 1, 1, bias=True, bn_eps=bn5),
                           conv(share_conv_channel, c, 3, 1, 1, bias=True, relu=False)))
            self.heads.append(hs)
        self._batched = None
        self.loaded = False  # parameters from a checkpoint (checkpoint.load_state_dict), not seeded

    def all_convs(self):
        out = self.trunk.convs() + [self.shared]
        for hs in self.heads:
            for _, a, b in hs:
                out += [a, b]
        return out

    def head_planes(self):
        """Output planes of the CenterHead: per task the common heads' channels (2 + 1 + 3 + 2 + 2 by default) + classes
        (70 for the six nuScenes tasks)."""
        return sum(sum(c for _, c in self.common_heads) + n for n in self.tasks)

    def head_flops(self, h, w):
        """Algorithmic flops (2 x MACs) of the CenterHead on an h x w map: the shared conv, the ConvModules and the output
        convs, and their sum "head"."""
        px = h * w
        sh = self.shared
        out = dict(head_shared=2.0 * px * sh.cin * sh.cout * sh.k * sh.k, head_convmodules=0.0, head_output=0.0)
        for hs in self.heads:
            for _, a, f in hs:
                out["head_convmodules"] += 2.0 * px * a.cin * a.cout * a.k * a.k
                out["head_output"] += 2.0 * px * f.cin * f.cout * f.k * f.k
        out["head"] = out["head_shared"] + out["head_convmodules"] + out["head_output"]
        return out

    def init_weight(self, seed=0, device="cuda", randomize_bn=False, bn_gain=1.0):
        """device=None: numpy parameters only (enough for export_numpy / the CPU arm).  bn_gain multiplies every BatchNorm
        gamma (sqrt(6) keeps the activations O(1) through the stack, see sparse_nn.BatchNorm.init_parameters)."""
        rng = np.random.default_rng(seed)
        hm_finals = {id(b) for hs in self.heads for name, _, b in hs if name == "hm"}
        finals = {id(b) for b in self.finals()}
        for c in self.all_convs():  # hm bias = -2.19 (center_head.py:113-117)
            # the 1-3 channel output convs have no per-conv image in f16 mode: they run in one tap-as-N launch
            dev = None if (self.f16 and id(c) in finals) else device
            c.init(rng, dev, randomize_bn, bias_value=-2.19 if id(c) in hm_finals else None, bn_gain=bn_gain)
        return self.derive(device)

    def finals(self):
        """The output convs: in f16 mode they have no per-conv device image (they run in one tap-as-N launch)."""
        return [f for hs in self.heads for _, _, f in hs]

    def derive(self, device):
        """The device state that is derived from the whole model's parameters (each conv's own image comes from
        _Conv.set_parameters): the permuted first conv of the (z, c) pixel input, and (on the next forward) the batched
        ConvModule conv and the tap-as-N output-conv images.  Called after new parameters, seeded or loaded."""
        self._batched = None
        self._first_zc = None
        # bev_depth 1 (pillars): the (z, c) order is the (c, z) order, the first conv reads the pixel rows as it is
        if self.f16 and device is not None and self.bev_depth > 1 and self.in_channels % self.bev_depth == 0:
            # second image of the first conv for BEV tensors that arrive as pixel fp16-pair rows straight from the sparse
            # rows (SparseCooTensor.to_pixel_h16): there a pixel's channels are ordered (z, c) = z * C + c, while the
            # reference's to_dense + transpose + reshape (sparse_resnet.py:202-206) orders them (c, z) = c * D + z.  The
            # input-channel axis of the weights is permuted once here instead of permuting activations every frame.
            c0 = self.blocks[0][0]
            D, C = self.bev_depth, self.in_channels // self.bev_depth
            perm = np.asarray([c * D + z for z in range(D) for c in range(C)])
            zc = _Conv(c0.cin, c0.cout, c0.k, c0.stride, c0.padding, bias=c0.has_bias, bn_eps=c0.bn_eps, relu=c0.relu, f16=True)
            zc.np = dict(c0.np, weight=np.ascontiguousarray(c0.np["weight"][:, perm]))
            zc.dev = dict(c0.dev, packed=dc.pack_conv_weight_f16(torch.from_numpy(zc.np["weight"]).to(device), zc.n_tile))
            self._first_zc = zc
        return self

    def export_numpy(self):
        return dict(self.trunk.export_numpy(), shared=self.shared.np,
                    heads=[[(n, a.np, b.np) for n, a, b in hs] for hs in self.heads])

    # ---- RPN + neck + shared conv: bev [B, C, H, W] fp32 -> (pixel rows of the shared feature map, its shape)
    def _trunk(self, bev, shape=None):
        """bev: fp32 NCHW tensor, or (shape given) pixel fp16-pair rows [B*H*W, 2*C] with shape = (B, H, W, C)."""
        first = None
        if shape is None:
            b, c, h, w = bev.shape
            x = dc.nchw_to_pixel_h16(bev) if self.f16 else dc.nchw_to_pixel_split(bev)
            shape = (b, h, w, c)
        else:
            if not self.f16 or (self.bev_depth > 1 and self._first_zc is None):
                raise ValueError("pixel fp16-pair input needs the f16 head")
            x = bev
            first = self._first_zc  # channels arrive in (z, c) order (None with bev_depth 1: the trunk's own first conv)
        cat, (b, H, W, _) = self.trunk(x, shape, first=first)
        s, _, _ = self.shared(cat, (b, H, W, self.fpn_channels))
        return s, (b, H, W, self.shared.cout)

    def _final_convs(self, mid, shape, in_C, groups_params, planes_total, device):
        """Grouped 64 -> {1..3} output convs in one launch: tensor cores with the 9 taps in the GEMM's N dimension on the
        fp16-pair path (p3d_head_out_conv_f16), CUDA cores (p3d_head_final_conv) on the tf32 one."""
        from ._lib import check, lib
        from ._mem import ptr, stream
        b, H, W, cin = shape
        gp = groups_params
        planes = torch.empty((b, planes_total, H, W), dtype=torch.float32, device=device)
        if self.f16:
            check(lib().p3d_head_out_conv_f16(ptr(mid), b, H, W, in_C, cin, int(gp["cnt9"].numel()), ptr(gp["packed9"]),
                                              ptr(gp["bias9"]), ptr(gp["cin0_9"]), ptr(gp["plane0_9"]), ptr(gp["cnt9"]),
                                              planes_total, ptr(planes), stream(device)), "head_out_conv_f16")
        else:
            check(lib().p3d_head_final_conv(ptr(mid), b, H, W, in_C, cin, len(gp["cnt"]), ptr(gp["fw"]), ptr(gp["fb"]),
                                            gp["plane0"].ctypes.data, gp["cnt"].ctypes.data, planes_total, ptr(planes),
                                            stream(device)), "head_final_conv")
        return planes

    def _group_params(self, finals, cin, device):
        """Weights of a list of output convs [(name, _Conv)] in the grouped form of _final_convs: on the fp16-pair path
        per (virtual) group the tap-as-N weight image W2[c][tap * 3 + co] + bias [4]; on the tf32 one [groups][9][Cin][4]
        fp32 + bias [groups][4] for the CUDA-core kernel."""
        groups = len(finals)
        wts, plane0, cnt, p0 = [], [], [], 0
        for _, f in finals:
            wts.append(f.np["weight"].transpose(2, 3, 1, 0).reshape(9, cin, f.cout))  # [k, cin, 3, 3] -> [tap][cin][k]
            plane0.append(p0)
            cnt.append(f.cout)
            p0 += f.cout
        out = dict(plane0=np.asarray(plane0, np.int32), cnt=np.asarray(cnt, np.int32), planes=p0)
        if not self.f16:
            fw = np.zeros((groups, 9, cin, 4), np.float32)
            fb = np.zeros((groups, 4), np.float32)
            for g, (_, f) in enumerate(finals):
                fw[g, :, :, :f.cout] = wts[g]
                fb[g, :f.cout] = f.np["bias"]
            out.update(fw=torch.from_numpy(fw).to(device), fb=torch.from_numpy(fb).to(device))
            return out
        from ._lib import check, lib
        from ._mem import ptr, stream
        L = lib()
        # tap-as-N form (p3d_head_out_conv_f16): W2[c][tap * 3 + j]; a conv with more than 3 output channels becomes
        # several virtual groups over the same input slice
        w9, b9, cin0, pl0, cn = [], [], [], [], []
        for g, (_, f) in enumerate(finals):
            for j0 in range(0, f.cout, 3):
                k = min(3, f.cout - j0)
                w27 = np.zeros((cin, 9, 3), np.float32)
                w27[:, :, :k] = wts[g][:, :, j0:j0 + k].transpose(1, 0, 2)  # [tap][c][j] -> [c][tap][j]
                w2 = np.zeros((cin, 32), np.float32)
                w2[:, :27] = w27.reshape(cin, 27)
                bb = np.zeros((4,), np.float32)
                bb[:k] = f.np["bias"][j0:j0 + k]
                w9.append(w2)
                b9.append(bb)
                cin0.append(g * cin)
                pl0.append(int(plane0[g]) + j0)
                cn.append(k)
        blk9 = cin * 32 * 4
        packed9 = torch.zeros((len(w9) * blk9,), dtype=torch.uint8, device=device)
        for v, w2 in enumerate(w9):
            wt = torch.from_numpy(w2).to(device)
            check(L.p3d_dense_conv2d_f16_pack_weights(ptr(wt), 1, cin, 32, ptr(packed9[v * blk9:(v + 1) * blk9]),
                                                      ptr(dc._status(device)), stream(device)), "pack_weights")
        i32 = lambda a: torch.from_numpy(np.asarray(a, np.int32)).to(device)  # noqa: E731
        out.update(packed9=packed9, bias9=torch.from_numpy(np.stack(b9)).to(device), cin0_9=i32(cin0), plane0_9=i32(pl0),
                   cnt9=i32(cn))
        return out

    def _batched_params(self, device):
        """One Conv(64 -> 36 * 64) with the 36 ConvModules' weights / folded BN concatenated along Cout, and the grouped
        form of the 36 output convs (_group_params)."""
        if self._batched is not None:
            return self._batched
        firsts = [a for hs in self.heads for _, a, _ in hs]
        finals = [(n, f) for hs in self.heads for n, _, f in hs]
        cin = firsts[0].cin
        big = _Conv(cin, sum(a.cout for a in firsts), 3, 1, 1, bias=True, bn_eps=firsts[0].bn_eps, f16=self.f16)
        w = np.concatenate([a.np["weight"] for a in firsts], 0)
        scale, shift = [], []
        for a in firsts:  # same folding as _Conv.init
            bn = a.np["bn"]
            s_ = bn["gamma"].astype(np.float64) / np.sqrt(bn["var"].astype(np.float64) + bn["eps"])
            scale.append(s_)
            shift.append((a.np["bias"].astype(np.float64) - bn["mean"]) * s_ + bn["beta"])
        pack = dc.pack_conv_weight_f16 if self.f16 else dc.pack_conv_weight
        big.dev = dict(packed=pack(torch.from_numpy(w).to(device), big.n_tile),
                       scale=torch.from_numpy(np.concatenate(scale).astype(np.float32)).to(device),
                       shift=torch.from_numpy(np.concatenate(shift).astype(np.float32)).to(device))
        self._batched = dict(big=big, names=[n for n, _ in finals])
        self._batched.update(self._group_params(finals, cin, device))
        return self._batched

    def calibrate_heatmap_bias(self, bev, score_threshold=0.1, target_frac=0.014, shape=None):
        """Seeded random weights give heat maps that hover around the initial bias (sigmoid(-2.19) = 0.1: half of all cells
        would pass a 0.1 score threshold, 16k candidates per task).  A trained CenterPoint fires on a few hundred cells per
        task; SURVEY.md §8d specifies ~1.4 % of cells above the threshold for the synthetic workload.  This shifts the bias of
        every task's heat-map conv so that `target_frac` of the cells of `bev`'s frame score above `score_threshold`
        (weights stay seeded and are exported unchanged to the CPU arm).  bev: as forward() takes it (with `shape`, pixel
        fp16-pair rows)."""
        if self.loaded:
            raise RuntimeError("calibrate_heatmap_bias moves the heat-map biases of seeded random weights; this head's "
                               "weights were loaded from a checkpoint and are kept as trained")
        out = self.forward(bev, shape)
        logit_thr = float(np.log(score_threshold / (1.0 - score_threshold)))
        for t, hs in enumerate(self.heads):
            hm = out["hm"][t].float().amax(dim=1).flatten()
            k = max(1, int(round(hm.numel() * (1.0 - target_frac))))
            q = float(torch.kthvalue(hm, k).values.item())
            fin = [f for name, _, f in hs if name == "hm"][0]
            fin.np["bias"] = (fin.np["bias"] + np.float32(logit_thr - q)).astype(np.float32)
        self._batched = None
        return self

    def forward_h16(self, rows, shape):
        """Same as forward() for a BEV given as pixel fp16-pair rows (SparseResNet3D.forward(pixel_h16=True))."""
        return self.forward(rows, shape)

    def fused_heads(self, bp):
        """Whether forward fuses the output convs' tap-as-N GEMM into the batched ConvModule conv (p3d_head_conv_p_f16,
        then p3d_head_tap_sum): fp16-pair path, 64-channel heads on the 128-wide N tile (two heads per tile), and every
        output conv <= 3 channels, so that each head is one tap-as-N group.  Otherwise the heads' image is written and
        read back by p3d_head_out_conv_f16."""
        big = bp["big"]
        return (self.f16 and self.shared.cout == 64 and big.n_tile == 128 and big.cout % 128 == 0
                and all(int(k) <= 3 for k in bp["cnt"]))

    def _heads_conv_p(self, s, shape, bp, device):
        """Fused path, first launch: the batched ConvModule conv and the output convs' per-pixel GEMM -> P
        [B, heads, H, W, 28] fp32 (the heads' 64-channel image is never written)."""
        from ._lib import check, lib
        from ._mem import ptr, stream
        b, H, W, cin = shape
        big = bp["big"]
        d = big.dev
        p = torch.empty((b, big.cout // 64, H, W, 28), dtype=torch.float32, device=device)
        check(lib().p3d_head_conv_p_f16(ptr(s), b, H, W, cin, ptr(d["packed"]), big.cout, ptr(d["scale"]), ptr(d["shift"]),
                                        ptr(bp["packed9"]), ptr(p), ptr(dc._status(device)), stream(device)), "head_conv_p_f16")
        return p

    def _tap_sum(self, p, bp, device):
        """Fused path, second launch: P -> the output convs' fp32 planes [B, planes, H, W]."""
        from ._lib import check, lib
        from ._mem import ptr, stream
        b, groups, H, W, _ = p.shape
        planes = torch.empty((b, bp["planes"], H, W), dtype=torch.float32, device=device)
        check(lib().p3d_head_tap_sum(ptr(p), b, H, W, groups, ptr(bp["bias9"]), ptr(bp["plane0_9"]), ptr(bp["cnt9"]),
                                     bp["planes"], ptr(planes), stream(device)), "head_tap_sum")
        return planes

    def forward(self, bev, shape=None):
        """bev [B, C, H, W] fp32 -> dict name -> list (per task) of [B, k, H, W] fp32 tensors.  The 36 ConvModules run as
        one 64 -> 2304 convolution, the 36 output convs as one grouped launch (fused_heads: the conv also runs the
        output convs' GEMM, and one launch sums its taps)."""
        s, shape = self._trunk(bev, shape)
        bp = self._batched_params(bev.device)
        big = bp["big"]
        if self.fused_heads(bp):
            planes = self._tap_sum(self._heads_conv_p(s, shape, bp, bev.device), bp, bev.device)
        else:
            mid, _, _ = big(s, shape)  # [B*H*W] pixel rows of 36 * 64 channels
            planes = self._final_convs(mid, shape, big.cout, bp, bp["planes"], bev.device)
        out = {}
        for name, p0, k in zip(bp["names"], bp["plane0"], bp["cnt"]):
            out.setdefault(name, []).append(planes[:, int(p0):int(p0) + int(k)])
        return out

    __call__ = forward
    forward_batched = forward

    def forward_per_head(self, bev):
        """Layer-by-layer form (72 launches for the heads), kept for the parity tests: same result as forward()."""
        s, shape = self._trunk(bev)
        out = {}
        for hs in self.heads:
            for name, a, fin in hs:
                t, _, _ = a(s, shape)
                k, cin = fin.cout, fin.cin
                if self.f16:
                    gp = self._group_params([(name, fin)], cin, bev.device)
                    planes = self._final_convs(t, shape, a.cout, gp, k, bev.device)
                else:
                    _, planes, _ = fin(t, shape, want_nchw=True)
                out.setdefault(name, []).append(planes)
        return out

    # ---- CenterHead.predict_by_custom_op (center_head.py:294-339, SURVEY §8a-14): marshal the per-task head tensors
    def predict_by_custom_op(self, example, preds_dicts, test_cfg, **kwargs):
        """Same positional order as the reference (called as predict_by_custom_op(samples, preds, self.test_cfg),
        centerpoint.py:163,177).  preds_dicts: the reference's list of per-task dicts, or forward()'s dict
        name -> [tensor per task].  test_cfg: mapping or attribute object with the yml's keys; the NMS settings are read
        from the nested `nms` section like the reference (test_cfg.nms.nms_iou_threshold ...) and, failing that, from flat
        keys.  Returns the reference's one-element list of {meta, box3d_lidar, label_preds, scores}."""
        postprocess_fn = kwargs.get("postprocess_fn")
        if postprocess_fn is None:
            from .ops.centerpoint_postprocess import centerpoint_postprocess as postprocess_fn

        def get(obj, key):
            return obj[key] if isinstance(obj, dict) else getattr(obj, key)

        def has(obj, key):
            return key in obj if isinstance(obj, dict) else hasattr(obj, key)

        nms = get(test_cfg, "nms") if has(test_cfg, "nms") else test_cfg
        if isinstance(preds_dicts, dict):
            preds_dicts = [{k: v[t] for k, v in preds_dicts.items()} for t in range(len(self.tasks))]
        hm, reg, height, dim, vel, rot, num_classes, flag = [], [], [], [], [], [], [], 0
        for task_id, pd in enumerate(preds_dicts):
            for nc in self.num_classes:  # as in the reference the list grows to T*T entries; the op reads the first T
                num_classes.append(flag)
                flag += nc
            hm.append(pd["hm"])
            reg.append(pd["reg"])
            height.append(pd["height"])
            dim.append(pd["dim"])
            vel.append(pd["vel"] if self.with_velocity else pd["reg"])
            rot.append(pd["rot"])
        bboxes, scores, labels = postprocess_fn(
            hm, reg, height, dim, vel, rot, get(test_cfg, "voxel_size"), get(test_cfg, "point_cloud_range"),
            get(test_cfg, "post_center_limit_range"), num_classes, get(test_cfg, "down_ratio"),
            get(test_cfg, "score_threshold"), get(nms, "nms_iou_threshold"), get(nms, "nms_pre_max_size"),
            get(nms, "nms_post_max_size"), self.with_velocity)
        meta = None if (not example or "meta" not in example or len(example["meta"]) == 0) else example["meta"][0]
        return [{"meta": meta, "box3d_lidar": bboxes, "label_preds": labels, "scores": scores}]
