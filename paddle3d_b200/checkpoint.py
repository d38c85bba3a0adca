"""Trained Paddle3D parameters for the LiDAR models: read a `.pdparams` file and map its names onto this repository's layers.

    read_pdparams(path)                 the file's {structured name: float32 ndarray}, read without running its code
    centerpoint_voxel(net, dense)       name tables: one list of parameter groups per model, the only place that knows
    centerpoint_pillars(model)          Paddle3D's names.  state_dict(table) reads the parameters under those names and
    pointpillars(model)                 in Paddle's layouts, load_state_dict(table, sd, device) checks and assigns them

`paddle.save(layer.state_dict(), path)` writes a pickle (protocol 4 in Paddle 2.x) of {structured name: numpy.ndarray}
plus a "StructuredToParameterName@@" entry (structured name -> the framework's parameter name); some 2.x versions store a
tensor as a (name, ndarray) tuple.  The file comes from outside the program, so it is never given to pickle.load: the
unpickler here resolves only the globals an ndarray and a dict need and refuses any other by name before calling it.

Layouts are Paddle's own, the ones the layers here keep: sparse Conv3D / SubmConv3D weight [kD, kH, kW, Cin, Cout],
Conv2D [Cout, Cin, kH, kW], Conv2DTranspose [Cin, Cout, kH, kW], Linear [in, out], BatchNorm weight / bias / _mean /
_variance [C].  Loading changes parameter values only: every device image (BN folds, packed tensor-core weights, the
first RPN conv's (z, c) image, the batched CenterHead conv, PointPillars' one cls | box | dir conv) is re-derived from
them by the same code that derives it from seeded parameters.

PARITY UNPINNED: the names are recalled, not checked against a Paddle3D checkout, from the module attributes of
    CenterPoint         paddle3d/models/detection/centerpoint/centerpoint.py: voxel_encoder, middle_encoder, backbone,
                        neck, bbox_head
    SparseResNet3D      paddle3d/models/middle_encoders/sparse_resnet.py: conv_input, conv1..conv4 (nn.Sequential of
                        Conv3D, BatchNorm, ReLU, then SparseBasicBlock conv1 / bn1 / conv2 / bn2), extra_conv
    PillarFeatureNet    paddle3d/models/voxel_encoders/pillar_encoder.py: pfn_layers.i.linear / .norm
    SecondBackbone      paddle3d/models/backbones/second_backbone.py: blocks.i, nn.Sequential (conv, BN, ReLU) x n
    SecondFPN           paddle3d/models/necks/second_fpn.py: deblocks.i, nn.Sequential (conv or deconv, BN, ReLU)
    CenterHead          paddle3d/models/heads/dense_heads/center_head.py: shared_conv (conv, BN, ReLU); tasks.t.<head>
                        of SeparateHead, nn.Sequential (conv, BN, ReLU, final conv)
    PointPillars        paddle3d/models/detection/pointpillars/pointpillars.py: pillar_encoder, backbone, neck, head;
                        its SSD head's cls_head / box_head / dir_head 1x1 convs (mmdet3d's Anchor3DHead names them
                        conv_cls / conv_box / conv_dir_cls)
A checkout corrects the table functions below and nothing else."""
import collections
import io
import os
import pickle

import numpy as np
import torch

STRUCTURED_NAMES = "StructuredToParameterName@@"

# the globals a pickled {name: ndarray} (or OrderedDict) needs, and nothing else
_ALLOWED = {("numpy.core.multiarray", "_reconstruct"), ("numpy._core.multiarray", "_reconstruct"),
            ("numpy", "ndarray"), ("numpy", "dtype"), ("collections", "OrderedDict")}


class _Unpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if (module, name) not in _ALLOWED:
            raise pickle.UnpicklingError("refusing global %s.%s in a .pdparams file: only numpy arrays and a dict are "
                                         "allowed" % (module, name))
        return super().find_class(module, name)


def _check_array(key, a):
    """float32 (finite) or integer: the dtypes a parameter file holds."""
    if not isinstance(a, np.ndarray):
        raise ValueError("%s: not an array (%s)" % (key, type(a).__name__))
    if a.dtype.kind in "iub":
        return
    if a.dtype != np.float32:
        raise ValueError("%s: dtype %s; only float32 parameters are read (fp16 / fp64 checkpoints are not)" % (key, a.dtype))
    if not np.isfinite(a).all():
        raise ValueError("%s: non-finite values" % key)


def read_pdparams(path):
    """A `.pdparams` file (a path, or a binary file object) -> {structured name: ndarray}: float32 parameters and any
    integer entries as stored, the (name, ndarray) tuple form unwrapped, the StructuredToParameterName@@ entry dropped.
    Raises pickle.UnpicklingError for any global other than an ndarray's or a dict's, ValueError (naming the key) for a
    value that is not a float32 or integer array or holds a non-finite value."""
    if isinstance(path, (str, os.PathLike)):
        with open(path, "rb") as f:
            obj = _Unpickler(io.BytesIO(f.read())).load()
    else:
        obj = _Unpickler(path).load()
    if not isinstance(obj, dict):
        raise ValueError("%s: expected a dict of parameters, got %s" % (path, type(obj).__name__))
    out = collections.OrderedDict()
    for k, v in obj.items():
        if k == STRUCTURED_NAMES:
            continue
        if isinstance(v, tuple) and len(v) == 2 and isinstance(v[1], np.ndarray):
            v = v[1]
        _check_array(k, v)
        out[k] = v
    return out


def as_state_dict(weights):
    """weights: a `.pdparams` path or an already read state dict."""
    return read_pdparams(weights) if isinstance(weights, (str, os.PathLike)) else weights


# ---------------------------------------------------------------------------------------------------- parameter groups
# A group is one layer's parameters: shapes() {name: shape} from the layer's architecture (so a model that was never
# initialised can be loaded), get() {name: ndarray} of the current values, set(values, device) assigns and derives.
def _np(t):
    return np.ascontiguousarray(t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else t, np.float32)


class _SparseConv:
    def __init__(self, prefix, layer):
        self.p, self.l = prefix, layer

    def shapes(self):
        l = self.l
        out = {self.p + "weight": tuple(l.kernel_size) + (l.in_channels, l.out_channels)}
        if l.bias is not None:
            out[self.p + "bias"] = (l.out_channels,)
        return out

    def get(self):
        return {self.p + "weight": _np(self.l.weight), **({self.p + "bias": _np(self.l.bias)} if self.l.bias is not None
                                                         else {})}

    def set(self, v, device):
        b = v.get(self.p + "bias")
        self.l.assign_parameters(torch.from_numpy(v[self.p + "weight"]).to(device),
                                 None if b is None else torch.from_numpy(b).to(device))


_BN_NAMES = (("weight", "gamma"), ("bias", "beta"), ("_mean", "mean"), ("_variance", "var"))


class _SparseBN:
    def __init__(self, prefix, layer):
        self.p, self.l = prefix, layer

    def shapes(self):
        return {self.p + n: (self.l.num_features,) for n, _ in _BN_NAMES}

    def get(self):
        l = self.l
        return {self.p + n: _np(t) for n, t in zip(("weight", "bias", "_mean", "_variance"),
                                                   (l.weight, l.bias, l._mean, l._variance))}

    def set(self, v, device):
        self.l.set_parameters(*[torch.from_numpy(v[self.p + n]).to(device) for n, _ in _BN_NAMES])


class _DenseConv:
    """A dense_head._Conv: the conv under `conv` (weight, bias if it has one), its BatchNorm under `bn` (if it has one).
    packed=False: the conv has no device image of its own (the CenterHead's output convs on the fp16-pair path)."""

    def __init__(self, conv, bn, layer, packed=True):
        self.c, self.b, self.l, self.packed = conv, bn, layer, packed

    def shapes(self):
        l = self.l
        out = {self.c + "weight": l.weight_shape()}
        if l.has_bias:
            out[self.c + "bias"] = (l.cout,)
        if l.bn_eps is not None:
            out.update({self.b + n: (l.cout,) for n, _ in _BN_NAMES})
        return out

    def get(self):
        p = self.l.np
        out = {self.c + "weight": _np(p["weight"])}
        if self.l.has_bias:
            out[self.c + "bias"] = _np(p["bias"])
        if self.l.bn_eps is not None:
            out.update({self.b + n: _np(p["bn"][f]) for n, f in _BN_NAMES})
        return out

    def set(self, v, device):
        bn = {f: v[self.b + n] for n, f in _BN_NAMES} if self.l.bn_eps is not None else None
        self.l.set_parameters(v[self.c + "weight"], v.get(self.c + "bias"), bn, device if self.packed else None)


class _PFN:
    """One PFNLayer (Linear [in, out] without bias, BatchNorm1D) held as a dict weight / gamma / beta / mean / var / eps."""

    def __init__(self, prefix, d, shape):
        self.p, self.d, self.shape = prefix, d, tuple(shape)

    def shapes(self):
        return {self.p + "linear.weight": self.shape, **{self.p + "norm." + n: (self.shape[1],) for n, _ in _BN_NAMES}}

    def get(self):
        return {self.p + "linear.weight": _np(self.d["weight"]),
                **{self.p + "norm." + n: _np(self.d[f]) for n, f in _BN_NAMES}}

    def set(self, v, device):
        self.d.update(weight=v[self.p + "linear.weight"], **{f: v[self.p + "norm." + n] for n, f in _BN_NAMES})


class _SplitConv:
    """One 1x1 conv with bias (`layer`) whose output channels are the concatenation of several Paddle convs:
    parts [(prefix, channels)] in channel order."""

    def __init__(self, parts, layer):
        self.parts, self.l = parts, layer

    def shapes(self):
        out = {}
        for p, n in self.parts:
            out.update({p + "weight": (n, self.l.cin, 1, 1), p + "bias": (n,)})
        return out

    def get(self):
        w, b = self.l.np["weight"], self.l.np["bias"]
        out, c0 = {}, 0
        for p, n in self.parts:
            out.update({p + "weight": _np(w[c0:c0 + n]), p + "bias": _np(b[c0:c0 + n])})
            c0 += n
        return out

    def set(self, v, device):
        w = np.concatenate([v[p + "weight"] for p, _ in self.parts], 0)
        b = np.concatenate([v[p + "bias"] for p, _ in self.parts], 0)
        self.l.set_parameters(w, b, None, device)


# ---------------------------------------------------------------------------------------------------- name tables
def _sparse_resnet3d(p, net):
    """layers.SparseResNet3D: conv_input, conv1 (2 blocks), conv2..conv4 (strided conv, BN, ReLU, 2 blocks), extra_conv."""
    def blocks(q, bs, first):
        out = []
        for j, b in enumerate(bs):
            r = "%s%d." % (q, first + j)
            out += [_SparseConv(r + "conv1.", b.conv1), _SparseBN(r + "bn1.", b.bn1),
                    _SparseConv(r + "conv2.", b.conv2), _SparseBN(r + "bn2.", b.bn2)]
        return out
    g = [_SparseConv(p + "conv_input.0.", net.conv_input[0]), _SparseBN(p + "conv_input.1.", net.conv_input[1])]
    g += blocks(p + "conv1.", net.blocks0, 0)
    for i, (down, bs) in enumerate(net.stages):
        q = "%sconv%d." % (p, i + 2)
        g += [_SparseConv(q + "0.", down[0]), _SparseBN(q + "1.", down[1])] + blocks(q, bs, 3)
    g += [_SparseConv(p + "extra_conv.0.", net.extra_conv[0]), _SparseBN(p + "extra_conv.1.", net.extra_conv[1])]
    return g


def _second_trunk(blocks, deblocks):
    """SecondBackbone blocks (conv j at index 3 j, its BN at 3 j + 1) and SecondFPN deblocks (conv 0, BN 1)."""
    g = []
    for i, blk in enumerate(blocks):
        for j, c in enumerate(blk):
            g.append(_DenseConv("backbone.blocks.%d.%d." % (i, 3 * j), "backbone.blocks.%d.%d." % (i, 3 * j + 1), c))
    for i, de in enumerate(deblocks):
        g.append(_DenseConv("neck.deblocks.%d.0." % i, "neck.deblocks.%d.1." % i, de))
    return g


def _center_head(dense):
    """dense_head.DenseRPNHead: trunk, then CenterHead shared_conv and per task the SeparateHead of each head."""
    g = _second_trunk(dense.blocks, dense.deblocks)
    g.append(_DenseConv("bbox_head.shared_conv.0.", "bbox_head.shared_conv.1.", dense.shared))
    for t, hs in enumerate(dense.heads):
        for name, a, f in hs:
            q = "bbox_head.tasks.%d.%s." % (t, name)
            g += [_DenseConv(q + "0.", q + "1.", a), _DenseConv(q + "3.", None, f, packed=not dense.f16)]
    return g


def centerpoint_voxel(net, dense):
    """CenterPoint-voxel (pipeline.CenterPointHotPath with with_head=True): SparseResNet3D and the DenseRPNHead."""
    return _sparse_resnet3d("middle_encoder.", net) + _center_head(dense)


def centerpoint_pillars(model):
    """centerpoint_pillars.CenterPointPillars: the two-layer PillarFeatureNet and the DenseRPNHead."""
    return ([_PFN("voxel_encoder.pfn_layers.%d." % i, d, s) for i, (d, s) in enumerate(zip(model.pfn, model.pfn_shapes()))]
            + _center_head(model.head))


def pointpillars(model):
    """pointpillars.PointPillars (car and cyclist / pedestrian): PillarFeatureNet, trunk, SSD head."""
    names = dict(cls="head.cls_head.", box="head.box_head.", dir="head.dir_head.")
    return ([_PFN("pillar_encoder.pfn_layers.0.", model.pfn, (model.F + 5, model.C))]
            + _second_trunk(model.trunk.blocks, model.trunk.deblocks)
            + [_SplitConv([(names[k], n) for k, n in model.head_splits()], model.head)])


# ---------------------------------------------------------------------------------------------------- both directions
def state_dict(table):
    """{Paddle3D name: float32 ndarray (a copy)} of a model's current parameters."""
    out = collections.OrderedDict()
    for g in table:
        out.update(g.get())
    return out


def load_state_dict(table, sd, device):
    """Check every entry of sd against the table, then assign them all (device: where the layers' device images go;
    None: numpy parameters only, for the models that keep them).  Missing names, unexpected float names, wrong shapes,
    dtypes other than float32 and non-finite values are reported together in one ValueError, raised before anything is
    assigned.  Integer entries outside the table are ignored (they are not parameters)."""
    expected = collections.OrderedDict()
    for g in table:
        expected.update(g.shapes())
    errors = []
    missing = [k for k in expected if k not in sd]
    if missing:
        errors.append("missing keys: " + ", ".join(missing))
    unexpected = [k for k, v in sd.items() if k not in expected and k != STRUCTURED_NAMES
                  and not (isinstance(v, np.ndarray) and v.dtype.kind in "iub")]
    if unexpected:
        errors.append("unexpected keys: " + ", ".join(unexpected))
    values = {}
    for k, shape in expected.items():
        if k not in sd:
            continue
        a = sd[k]
        try:
            _check_array(k, a)
            if a.dtype != np.float32:
                raise ValueError("%s: dtype %s, expected float32" % (k, a.dtype))
        except ValueError as e:
            errors.append(str(e))
            continue
        if tuple(a.shape) != tuple(shape):
            errors.append("%s: shape %s, expected %s" % (k, tuple(a.shape), tuple(shape)))
            continue
        values[k] = np.array(a, np.float32, copy=True, order="C")
    if errors:
        raise ValueError("state dict does not fit the model:\n  " + "\n  ".join(errors))
    for g in table:
        g.set(values, device)
