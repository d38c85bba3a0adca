"""Drop-in mirror of the `paddle.sparse` surface used by SparseResNet3D / SparseNet3D
(paddle3d/models/middle_encoders/sparse_resnet.py:22-23,31-60,84-111,125-206; sparsenet.py:38-52):

    nn.SubmConv3D(in, out, kernel_size, stride=1, padding=0, bias_attr=None, key=None)
    nn.Conv3D(in, out, kernel_size, stride=1, padding=0, bias_attr=None)
    nn.BatchNorm(num_features, momentum=0.9, epsilon=1e-5)     (inference statistics)
    nn.ReLU()
    sparse_coo_tensor(indices[4, nnz], values[nnz, C], shape), add(x, y), x.to_dense()

so the model file only changes its import line (`from paddle3d_b200.ops.sparse_nn import nn, ...`).

Execution model (GPU-first, not Paddle's): a convolution does not run when it is called.  It returns
a tensor with a *pending* fused kernel; BatchNorm / add / ReLU applied to that tensor fold into the
kernel's epilogue, and the single gather-GEMM launch happens when the values are needed (next conv,
to_dense, .values()).  conv -> bn -> relu, and conv -> bn -> add -> relu, are one launch each.
Row counts stay on the device (`num`), buffers are sized by capacity, no host sync anywhere.
"""
import math
import os

import numpy as np
import torch

from .._lib import check, host_ints, lib
from .._mem import ptr, require_cuda, stream, workspace
from . import pillar_scatter as _ps

# FP32         exact fp32 FMA on CUDA cores
# TF32X3       wgmma 3xTF32 on plain fp32 rows: the tf32 hi/lo split happens in the gather, once per gathering neighbour
# TF32X3_SPLIT wgmma 3xTF32 on split-layout rows [n][2][C]: whole-line cp.async gathers, split done once in the
#              producing layer's epilogue.  TF32X3 and TF32X3_SPLIT run the same kernel (csrc/sparse_conv_tc.cu); use
#              TF32X3_SPLIT for activations outside fp16's range
# F16X3        wgmma on fp16 hi/lo' pair rows (csrc/sparse_conv_f16.cu): same 22-bit products as TF32X3_SPLIT in half
#              the bytes, persistent + overlapped epilogue + device-chosen split-K; |activations| < 65504 (flagged)
FP32, TF32X3, TF32X3_SPLIT, F16X3 = 0, 1, 2, 4
TF32X3_TMA = TF32X3_SPLIT  # the name `bench.py --precision tf32x3_tma` selects
PRECISIONS = (FP32, TF32X3, TF32X3_SPLIT, F16X3)
ROWS_F32, ROWS_SPLIT, ROWS_H16 = 0, 1, 2  # activation layouts: [n, C] fp32 | [n][2][C] tf32 hi/lo | fp16 hi/lo' pairs
_default_precision = [FP32]
F16_MAX_SPLITS = 4
# F16X3 layers with (Cin, Cout) in {(16,16), (16,32), (32,32)} run on the register-gather warp-MMA kernel
# (csrc/sparse_conv_wm.cu: same rows, same arithmetic, missing neighbours are free); P3D_SPARSE_WM=0 keeps them on wgmma
NARROW_WM = [os.environ.get("P3D_SPARSE_WM", "1") != "0"]
_status = {}


def status_tensor(device):
    """Per-device int32 status word the fp16-pair kernels OR into (bit 0: value outside fp16's range was saturated)."""
    key = torch.device(device).index
    t = _status.get(key)
    if t is None:
        t = _status[key] = torch.zeros((1,), dtype=torch.int32, device=device)
    return t


def _check_precision(p):
    if p not in PRECISIONS:
        raise ValueError("unknown sparse conv precision %r (expected one of %s)" % (p, PRECISIONS))
    return p


def set_precision(p):
    """Default precision of the convs that do not set their own: FP32, TF32X3, TF32X3_SPLIT or F16X3."""
    _default_precision[0] = _check_precision(int(p))


def _triple(v):
    return [int(v)] * 3 if np.isscalar(v) else [int(x) for x in v]


def _rulebook_key(key, ksize):
    """Key of a SubM neighbour map in _IndexSet.subm_rulebooks: the layer's `key` (None: one map shared by the unkeyed
    layers) and kernel size."""
    return (key if key is not None else "_anon", tuple(ksize))


class _IndexSet:
    """Active sites of one resolution level: coords [cap, 4] (b, z, y, x), device count, its coordinate hash table
    (built once: from the coordinates for the input level, as a by-product of the site enumeration for the output of a
    strided conv) and the SubM rulebooks that share it."""

    def __init__(self, coords, num, cap, batch, spatial, table=None):
        self.coords, self.num, self.cap, self.batch, self.spatial = coords, num, cap, batch, list(spatial)
        self.subm_rulebooks = {}
        self.strided = {}      # id(Conv3D layer) -> (output _IndexSet, neighbour map), see _ConvBase.build_index
        self._table = table

    def table(self):
        if self._table is None:
            L = lib()
            dev = self.coords.device
            self._table = torch.empty((L.p3d_sparse_table_bytes(self.cap),), dtype=torch.uint8, device=dev)
            check(L.p3d_sparse_table_build(ptr(self.coords), ptr(self.num), self.cap, self.batch, host_ints(self.spatial),
                                           ptr(self._table), self._table.numel(), stream(dev)), "sparse_table_build")
        return self._table

    def subm_rulebook(self, ksize, key):
        k = _rulebook_key(key, ksize)
        nbr = self.subm_rulebooks.get(k)
        if nbr is None:
            K = ksize[0] * ksize[1] * ksize[2]
            dev = self.coords.device
            nbr = torch.empty((self.cap, K), dtype=torch.int32, device=dev)
            tab = self.table()
            check(lib().p3d_sparse_rulebook_subm_t(ptr(self.coords), ptr(self.num), self.cap, self.batch,
                                                   host_ints(self.spatial), host_ints(ksize), ptr(tab), tab.numel(),
                                                   ptr(nbr), stream(dev)), "sparse_rulebook_subm_t")
            self.subm_rulebooks[k] = nbr
        return nbr


class SparseCooTensor:
    def __init__(self, index, values=None, channels=None, pending=None):
        self.index = index
        self._vals = {ROWS_F32: values, ROWS_SPLIT: None, ROWS_H16: None}
        self._pending = pending
        self.channels = channels if channels is not None else values.shape[1]

    # ---- paddle-like surface
    @property
    def shape(self):
        return [self.index.batch] + self.index.spatial + [self.channels]

    def get(self, layout):
        """Row values in the requested layout; launches the pending fused kernel (asking it for this layout) or
        converts from the other layout with one small kernel."""
        v = self._vals[layout]
        if v is not None:
            return v
        if self._pending is not None:
            p, self._pending = self._pending, None
            _run(p, self, layout)
            v = self._vals[layout]
            if v is not None:
                return v
        f32 = self._vals[ROWS_F32]
        if f32 is None:  # materialise fp32 rows from whichever pair layout exists
            if self._vals[ROWS_H16] is not None:
                src = self._vals[ROWS_H16]
                f32 = torch.empty((self.index.cap, self.channels), dtype=torch.float32, device=src.device)
                check(lib().p3d_rows_convert_h16(ptr(src), 0, ptr(self.index.num), self.index.cap, self.channels, ptr(f32),
                                                 None, stream(src.device)), "rows_convert_h16")
            else:
                src = self._vals[ROWS_SPLIT]
                f32 = torch.empty((self.index.cap, self.channels), dtype=torch.float32, device=src.device)
                check(lib().p3d_rows_convert_layout(ptr(src), 1, ptr(self.index.num), self.index.cap, self.channels,
                                                    ptr(f32), stream(src.device)), "rows_convert_layout")
            self._vals[ROWS_F32] = f32
        if layout == ROWS_F32:
            return f32
        if layout == ROWS_H16:
            dst = torch.empty((self.index.cap, 2 * self.channels), dtype=torch.float16, device=f32.device)
            check(lib().p3d_rows_convert_h16(ptr(f32), 1, ptr(self.index.num), self.index.cap, self.channels, ptr(dst),
                                             ptr(status_tensor(f32.device)), stream(f32.device)), "rows_convert_h16")
        else:
            dst = torch.empty((self.index.cap, 2 * self.channels), dtype=torch.float32, device=f32.device)
            check(lib().p3d_rows_convert_layout(ptr(f32), 0, ptr(self.index.num), self.index.cap, self.channels, ptr(dst),
                                                stream(f32.device)), "rows_convert_layout")
        self._vals[layout] = dst
        return dst

    def values(self):
        return self.get(ROWS_F32)

    def indices(self):
        """[4, cap] like paddle (columns beyond nnz() are padding).  The output of a strided Conv3D lists its sites in
        first-appearance order (see Conv3D), not sorted as Paddle's does."""
        return self.index.coords.t()

    def nnz(self):
        return int(self.index.num[0].item()) if self.index.num is not None else self.index.cap

    def to_dense(self):
        """[B, D, H, W, C] (sparse_resnet.py:202).  SparseResNet3D's to_dense+transpose+reshape is served in one
        pass by `to_dense_bev`."""
        B = self.index.batch
        D, H, W = self.index.spatial
        return self.to_dense_bev().view(B, self.channels, D, H, W).permute(0, 2, 3, 4, 1)

    def to_dense_bev(self):
        return _ps.sparse_to_dense_bev(self.values(), self.index.coords, self.index.batch, self.index.spatial,
                                       num=self.index.num)

    def to_pixel_h16(self):
        """fp16-pair form of to_dense + transpose + reshape (sparse_resnet.py:202-206): pixel H16 rows
        [batch * ny * nx, 2 * D * C] float16 (channel = z * C + c) for the fp16-pair dense RPN - the rows of the last layer
        are scattered straight into it, no fp32 NCHW tensor is materialised."""
        rows = self.get(ROWS_H16)
        D, H, W = self.index.spatial
        B = self.index.batch
        out = torch.empty((B * H * W, 2 * D * self.channels), dtype=torch.float16, device=rows.device)
        check(lib().p3d_sparse_rows_to_pixel_h16(ptr(rows), ptr(self.index.coords), ptr(self.index.num), self.index.cap,
                                                 self.channels, B, D, H, W, ptr(out), stream(rows.device)),
              "sparse_rows_to_pixel_h16")
        return out, (B, H, W, D * self.channels)


def sparse_coo_tensor(indices, values, shape, stop_gradient=True, num=None):
    """indices [4, nnz] (paddle layout) or [nnz, 4]; values [nnz, C]; shape [B, D, H, W, C]."""
    values = require_cuda(values, "values", torch.float32)
    indices = require_cuda(indices, "indices")
    if indices.dim() != 2:
        raise ValueError("indices must be 2-D")
    if indices.shape[0] == 4 and indices.shape[1] != 4:
        indices = indices.t()
    coords = indices.to(torch.int32).contiguous()
    cap = coords.shape[0]
    idx = _IndexSet(coords, num, cap, int(shape[0]), [int(s) for s in shape[1:4]])
    return SparseCooTensor(idx, values=values, channels=int(shape[4]))


class _Pending:
    __slots__ = ("x", "nbr", "num", "cap", "K", "cin", "cout", "weight", "scale", "shift", "residual", "relu", "precision",
                 "wm")


PROFILE = None  # set to a list to record (cin, cout, K, precision, nbr, num, start_event, end_event, kernel) per conv launch


def _run(p, t, want):
    """Launch the fused gather-GEMM of pending `p` and store its result into tensor `t` (layout `want` when the
    kernel can produce it directly)."""
    L = lib()
    dev = p.nbr.device
    st = torch.cuda.current_stream(dev)
    if PROFILE is not None:
        s_ev, e_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if p.precision == F16X3:
        xin = p.x.get(ROWS_H16)
        res = p.residual.get(ROWS_H16) if p.residual is not None else None
        out_f32 = torch.empty((p.cap, p.cout), dtype=torch.float32, device=dev) if want != ROWS_H16 else None
        out_h16 = torch.empty((p.cap, 2 * p.cout), dtype=torch.float16, device=dev) if want == ROWS_H16 else None
        if PROFILE is not None:
            s_ev.record(st)
        if p.wm:
            wsb = L.p3d_sparse_conv_wm_workspace_bytes(p.cap, p.cout)
            # one scratch buffer per (capacity, channels): its head holds the self-cleaning stream-K tickets (zero on creation)
            ws = workspace(wsb, dev, "wm_streamk_%d_%d" % (p.cap, p.cout), zero=True)
            check(L.p3d_sparse_conv_wm(ptr(xin), ptr(p.nbr), ptr(p.num), p.cap, p.K, p.cin, p.cout, ptr(p.weight),
                                       ptr(p.scale), ptr(p.shift), ptr(res), int(p.relu), ptr(out_f32), ptr(out_h16),
                                       ptr(ws), wsb, ptr(status_tensor(dev)), stream(dev)), "sparse_conv_wm")
            t._vals[ROWS_F32], t._vals[ROWS_H16] = out_f32, out_h16
            if PROFILE is not None:
                e_ev.record(st)
                PROFILE.append((p.cin, p.cout, p.K, p.precision, p.nbr, p.num, s_ev, e_ev, "wm"))
            return
        wsb = L.p3d_sparse_conv_f16_workspace_bytes(p.cap, p.cout, F16_MAX_SPLITS)
        # one scratch buffer per (capacity, channels): its head holds the self-cleaning split-K tickets (zero on creation)
        ws = workspace(wsb, dev, "f16_splitk_%d_%d" % (p.cap, p.cout), zero=True) if wsb else None
        check(L.p3d_sparse_conv_f16(ptr(xin), ptr(p.nbr), ptr(p.num), p.cap, p.K, p.cin, p.cout, ptr(p.weight),
                                    ptr(p.scale), ptr(p.shift), ptr(res), int(p.relu), ptr(out_f32), ptr(out_h16),
                                    ptr(ws), wsb, F16_MAX_SPLITS, ptr(status_tensor(dev)), stream(dev)), "sparse_conv_f16")
        t._vals[ROWS_F32], t._vals[ROWS_H16] = out_f32, out_h16
    elif p.precision == TF32X3_SPLIT:
        xin = p.x.get(ROWS_SPLIT)
        res = p.residual.get(ROWS_SPLIT) if p.residual is not None else None
        # fp32 rows unless split rows are asked for: get() converts them to fp16-pair rows
        out_f32 = torch.empty((p.cap, p.cout), dtype=torch.float32, device=dev) if want != ROWS_SPLIT else None
        out_split = torch.empty((p.cap, 2 * p.cout), dtype=torch.float32, device=dev) if want == ROWS_SPLIT else None
        if PROFILE is not None:
            s_ev.record(st)
        wsb = L.p3d_sparse_conv_splitk_workspace_bytes(p.cap, p.cin, p.cout)  # > 0 for the wide (split-K) layers
        ws = workspace(wsb, dev, "splitk") if wsb else None
        check(L.p3d_sparse_conv_gather_gemm_split_ws(ptr(xin), ptr(p.nbr), ptr(p.num), p.cap, p.K, p.cin, p.cout,
                                                     ptr(p.weight), ptr(p.scale), ptr(p.shift), ptr(res), int(p.relu),
                                                     ptr(out_f32), ptr(out_split), ptr(ws), wsb, stream(dev)),
              "sparse_conv_gather_gemm_split_ws")
        t._vals[ROWS_F32], t._vals[ROWS_SPLIT] = out_f32, out_split
    elif (p.precision == FP32 and want == ROWS_H16 and p.residual is None and p.cin <= 8 and p.cout in (16, 32)
          and p.K * p.cin * p.cout * 4 <= 40 * 1024):
        # the few-channel input layer feeding fp16-pair layers: exact fp32 FMAs, pair rows written by the same kernel
        xin = p.x.get(ROWS_F32)
        out_h16 = torch.empty((p.cap, 2 * p.cout), dtype=torch.float16, device=dev)
        if PROFILE is not None:
            s_ev.record(st)
        check(L.p3d_sparse_conv_small_cin_h16(ptr(xin), ptr(p.nbr), ptr(p.num), p.cap, p.K, p.cin, p.cout, ptr(p.weight),
                                              ptr(p.scale), ptr(p.shift), int(p.relu), None, ptr(out_h16),
                                              ptr(status_tensor(dev)), stream(dev)), "sparse_conv_small_cin_h16")
        t._vals[ROWS_H16] = out_h16
    else:
        xin = p.x.get(ROWS_F32)
        res = p.residual.get(ROWS_F32) if p.residual is not None else None
        out = torch.empty((p.cap, p.cout), dtype=torch.float32, device=dev)
        if PROFILE is not None:
            s_ev.record(st)
        if p.precision == TF32X3:
            wsb = L.p3d_sparse_conv_splitk_workspace_bytes(p.cap, p.cin, p.cout)  # > 0 for the wide (split-K) layers
            ws = workspace(wsb, dev, "splitk") if wsb else None
            check(L.p3d_sparse_conv_gather_gemm_tf32x3_ws(ptr(xin), ptr(p.nbr), ptr(p.num), p.cap, p.K, p.cin, p.cout,
                                                          ptr(p.weight), ptr(p.scale), ptr(p.shift), ptr(res),
                                                          int(p.relu), ptr(out), ptr(ws), wsb, stream(dev)),
                  "sparse_conv_gather_gemm_tf32x3_ws")
        else:
            check(L.p3d_sparse_conv_gather_gemm(ptr(xin), ptr(p.nbr), ptr(p.num), p.cap, p.K, p.cin, p.cout,
                                                ptr(p.weight), ptr(p.scale), ptr(p.shift), ptr(res), int(p.relu), 0,
                                                ptr(out), stream(dev)), "sparse_conv_gather_gemm")
        t._vals[ROWS_F32] = out
    if PROFILE is not None:
        e_ev.record(st)
        PROFILE.append((p.cin, p.cout, p.K, p.precision, p.nbr, p.num, s_ev, e_ev, "tc"))


def _affine_act(x, scale, shift, residual, relu):
    v = x.values()
    out = torch.empty_like(v)
    res = residual.values() if residual is not None else None
    check(lib().p3d_sparse_affine_act(ptr(v), ptr(x.index.num), x.index.cap, x.channels, ptr(scale), ptr(shift),
                                      ptr(res), int(relu), ptr(out), stream(v.device)), "sparse_affine_act")
    return SparseCooTensor(x.index, values=out, channels=x.channels)


def _fuse(x, **changes):
    """A NEW lazy tensor whose pending kernel is x's with `changes` folded in.  x itself is left as it was (ADVICE r1: the
    fusing layers used to edit x._pending in place, so `y = relu(x)` also changed x and add() turned y into y + x for
    anyone still holding it); if x is consumed as well it simply launches its own, unfused kernel."""
    q = _Pending()
    for k in _Pending.__slots__:
        setattr(q, k, getattr(x._pending, k, None))
    for k, v in changes.items():
        setattr(q, k, v)
    return SparseCooTensor(x.index, channels=x.channels, pending=q)


def add(x, y):
    """paddle.sparse.add for tensors over the same index set (sparse_resnet.py:108)."""
    if x.index is not y.index:
        raise NotImplementedError("sparse add over different index sets is outside the hot path")
    p = x._pending
    if p is not None and p.residual is None and not p.relu:
        return _fuse(x, residual=y)
    p = y._pending
    if p is not None and p.residual is None and not p.relu:
        return _fuse(y, residual=x)
    return _affine_act(x, None, None, y, False)


class _Layer:
    training = False

    def __call__(self, *a, **k):
        return self.forward(*a, **k)

    def eval(self):
        return self


class _ConvBase(_Layer):
    subm = False

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 padding_mode="zeros", key=None, weight_attr=None, bias_attr=None, data_format="NDHWC"):
        if _triple(dilation) != [1, 1, 1] or groups != 1:
            raise NotImplementedError("dilation/groups are not used on the hot path")
        self.in_channels, self.out_channels = int(in_channels), int(out_channels)
        self.kernel_size, self.stride, self.padding = _triple(kernel_size), _triple(stride), _triple(padding)
        self.key = key
        self.weight = None  # [kD, kH, kW, Cin, Cout] fp32, Paddle's layout
        self.bias = None if bias_attr is False else "uninit"
        self.precision = None
        self.out_cap = None  # strided conv: capacity of the output index set (default 4x input capacity)

    def init_parameters(self, rng, device):
        """Kaiming-uniform(a=sqrt(5)) weights and uniform(+-1/sqrt(fan_in)) bias, as
        paddle3d.models.layers.param_init.reset_parameters (param_init.py:236-249) does for these layers."""
        kd, kh, kw = self.kernel_size
        fan_in = self.in_channels * kd * kh * kw
        bound = math.sqrt(6.0 / ((1 + 5.0) * fan_in))
        w = rng.uniform(-bound, bound, size=(kd, kh, kw, self.in_channels, self.out_channels)).astype(np.float32)
        self.weight = torch.from_numpy(w).to(device)
        if self.bias is not None:
            b = rng.uniform(-1 / math.sqrt(fan_in), 1 / math.sqrt(fan_in), size=(self.out_channels,)).astype(np.float32)
            self.bias = torch.from_numpy(b).to(device)
        return self

    def _packed_weight(self, K, f16=False, wm=False):
        """tf32 hi/lo (or fp16 hi/lo') shared-memory image of the weights, built once per layer (wm: the fragment-order
        image of the warp-MMA kernel)."""
        attr = "_packed_wm" if wm else "_packed_f16" if f16 else "_packed"
        pk = getattr(self, attr, None)
        if pk is None or pk[0] != self.weight.data_ptr():
            L = lib()
            dev = self.weight.device
            if wm:
                nbytes = L.p3d_sparse_conv_wm_packed_weight_bytes(K, self.in_channels, self.out_channels)
                buf = torch.empty((nbytes // 4,), dtype=torch.float32, device=dev)
                check(L.p3d_sparse_conv_wm_pack_weights(ptr(self.weight), K, self.in_channels, self.out_channels, ptr(buf),
                                                        ptr(status_tensor(dev)), stream(dev)), "sparse_conv_wm_pack_weights")
            elif f16:
                nbytes = L.p3d_sparse_conv_f16_packed_weight_bytes(K, self.in_channels, self.out_channels)
                buf = torch.empty((nbytes // 4,), dtype=torch.float32, device=dev)
                check(L.p3d_sparse_conv_f16_pack_weights(ptr(self.weight), K, self.in_channels, self.out_channels, ptr(buf),
                                                         ptr(status_tensor(dev)), stream(dev)), "sparse_conv_f16_pack_weights")
            else:
                nbytes = L.p3d_sparse_conv_packed_weight_bytes(K, self.in_channels, self.out_channels)
                buf = torch.empty((nbytes // 4,), dtype=torch.float32, device=dev)
                check(L.p3d_sparse_conv_pack_weights(ptr(self.weight), K, self.in_channels, self.out_channels, ptr(buf),
                                                     stream(dev)), "sparse_conv_pack_weights")
            pk = (self.weight.data_ptr(), buf)
            setattr(self, attr, pk)
        return pk[1]

    def set_parameters(self, weight, bias=None):
        self.weight = require_cuda(weight, "weight", torch.float32)
        self.bias = require_cuda(bias, "bias", torch.float32) if bias is not None else None
        return self

    def build_index(self, src):
        """Strided conv: output site set + neighbour map of `src` under this layer's geometry (cached on `src`)."""
        hit = src.strided.get(id(self))
        if hit is not None:
            return hit
        K = self.kernel_size[0] * self.kernel_size[1] * self.kernel_size[2]
        dev = src.coords.device
        cap = self.out_cap if self.out_cap is not None else 4 * src.cap
        out_coords = torch.empty((cap, 4), dtype=torch.int32, device=dev)
        n_out = torch.empty((4,), dtype=torch.int32, device=dev)
        nbr = torch.empty((cap, K), dtype=torch.int32, device=dev)
        L = lib()
        tab_in = src.table()
        tab_out = torch.empty((L.p3d_sparse_table_bytes(cap),), dtype=torch.uint8, device=dev)
        # fuse_subm = (ksize, key) of the SubM blocks that follow on the new level: their neighbour map comes out of the
        # same launch (p3d_sparse_rulebook_level_t) instead of a separate p3d_sparse_rulebook_subm_t call
        fuse = getattr(self, "fuse_subm", None)
        nbr_subm = sub_ks = None
        if fuse is not None:
            sub_ks = tuple(int(v) for v in fuse[0])
            nbr_subm = torch.empty((cap, sub_ks[0] * sub_ks[1] * sub_ks[2]), dtype=torch.int32, device=dev)
        check(L.p3d_sparse_rulebook_level_t(ptr(src.coords), ptr(src.num), src.cap, src.batch, host_ints(src.spatial),
                                            host_ints(self.kernel_size), host_ints(self.stride),
                                            host_ints(self.padding), ptr(tab_in), tab_in.numel(), ptr(out_coords),
                                            ptr(n_out), cap, ptr(tab_out), tab_out.numel(), ptr(nbr),
                                            host_ints(sub_ks) if sub_ks else None, ptr(nbr_subm), stream(dev)),
              "sparse_rulebook_level_t")
        osp = [(src.spatial[a] + 2 * self.padding[a] - self.kernel_size[a]) // self.stride[a] + 1 for a in range(3)]
        index = _IndexSet(out_coords, n_out, cap, src.batch, osp, table=tab_out)
        index.counters = n_out
        if nbr_subm is not None:
            index.subm_rulebooks[_rulebook_key(fuse[1], sub_ks)] = nbr_subm
        src.strided[id(self)] = (index, nbr)
        return index, nbr

    def forward(self, x):
        if self.weight is None or isinstance(self.bias, str):
            raise RuntimeError("conv parameters not set")
        K = self.kernel_size[0] * self.kernel_size[1] * self.kernel_size[2]
        p = _Pending()
        p.x, p.K, p.cin, p.cout = x, K, self.in_channels, self.out_channels
        p.weight, p.scale, p.shift, p.residual, p.relu = self.weight, None, self.bias, None, False
        p.wm = False
        p.precision = _check_precision(self.precision if self.precision is not None else _default_precision[0])
        if p.precision == F16X3:
            if not lib().p3d_sparse_conv_f16_packed_weight_bytes(K, self.in_channels, self.out_channels):
                p.precision = FP32  # e.g. the 5-channel input layer stays on the exact fp32 path
            elif NARROW_WM[0] and lib().p3d_sparse_conv_wm_packed_weight_bytes(K, self.in_channels, self.out_channels):
                p.wm = True
                p.weight = self._packed_weight(K, wm=True)
            else:
                p.weight = self._packed_weight(K, f16=True)
        elif p.precision in (TF32X3, TF32X3_SPLIT):
            if not lib().p3d_sparse_conv_packed_weight_bytes(K, self.in_channels, self.out_channels) or K > 32:
                p.precision = FP32  # e.g. the 5-channel input layer stays on the exact fp32 path
            else:
                p.weight = self._packed_weight(K)
        if self.subm:
            index = x.index
            p.nbr = index.subm_rulebook(self.kernel_size, self.key)
        else:
            index, p.nbr = self.build_index(x.index)
        p.num, p.cap = index.num, index.cap
        return SparseCooTensor(index, channels=self.out_channels, pending=p)


class SubmConv3D(_ConvBase):
    """Outputs only at the input sites; stride forced to 1 and padding to k//2 (Paddle's
    ResetSubmKernelSizeAndStrides)."""
    subm = True


class Conv3D(_ConvBase):
    """paddle.sparse.nn.Conv3D (strided).  The output's rows are its sites in first-appearance order: the input rows in
    row order and, within a row, the kernel taps in order k = (kz kH + ky) kW + kx, each site listed the first time one
    of them generates it.  The order depends only on the input index set, so the same input gives the same rows and the
    same bits in every run; Paddle's returns the sites sorted by linear key instead.  Of input rows sharing a coordinate
    the last stands for it; rows outside the grid generate no sites."""
    subm = False


class BatchNorm(_Layer):
    """paddle.sparse.nn.BatchNorm in inference mode: per-channel affine on the values."""

    def __init__(self, num_features, momentum=0.9, epsilon=1e-5, weight_attr=None, bias_attr=None,
                 data_format="NDHWC", use_global_stats=None):
        self.num_features, self.epsilon = int(num_features), float(epsilon)
        self.weight = self.bias = self._mean = self._variance = None
        self._folded = None
        self._bias_fold = {}  # conv bias tensor id -> folded shift (computed once, not per forward)

    def init_parameters(self, rng, device, randomize=False, gain=1.0):
        """gain: multiplies gamma.  The reference's fresh initialisation (gamma 1 after uniform(+-1/sqrt(fan_in)) weights)
        shrinks the activations by ~6x per conv + ReLU; sqrt(6) keeps them O(1) through the stack, which is the regime a
        trained network runs in and the one in which an end-to-end parity check says something."""
        c = self.num_features
        if randomize:  # non-trivial statistics for tests
            g, b = rng.uniform(0.5, 1.5, c), rng.uniform(-0.2, 0.2, c)
            m, v = rng.uniform(-0.1, 0.1, c), rng.uniform(0.5, 1.5, c)
        else:  # constant_init(weight, 1), constant_init(bias, 0), running stats (0, 1): sparse_resnet.py:177-183
            g, b, m, v = np.ones(c), np.zeros(c), np.zeros(c), np.ones(c)
        g = g * gain
        return self.set_parameters(*[torch.from_numpy(np.asarray(a, np.float32)).to(device) for a in (g, b, m, v)])

    def set_parameters(self, weight, bias, mean, variance):
        self.weight, self.bias, self._mean, self._variance = weight, bias, mean, variance
        # fold once, in fp64 on the host side of the parameters (tiny): y = x*scale + shift
        w, b, m, v = [t.double() for t in (weight, bias, mean, variance)]
        scale = w / torch.sqrt(v + self.epsilon)
        self._folded = (scale.float().contiguous(), (b - m * scale).float().contiguous())
        return self

    def forward(self, x):
        scale, shift = self._folded
        p = x._pending
        if p is not None and p.scale is None and p.residual is None and not p.relu:
            # (conv + bias) * scale + shift  ==  conv * scale + (bias * scale + shift)
            if p.shift is not None:
                key = p.shift.data_ptr()
                if key not in self._bias_fold:
                    self._bias_fold[key] = (p.shift.double() * scale.double() + shift.double()).float().contiguous()
                shift = self._bias_fold[key]
            return _fuse(x, shift=shift, scale=scale)
        return _affine_act(x, scale, shift, None, False)


class ReLU(_Layer):
    def forward(self, x):
        p = x._pending
        if p is not None:
            return _fuse(x, relu=True)
        return _affine_act(x, None, None, None, True)


class _NN:
    SubmConv3D, Conv3D, BatchNorm, ReLU = SubmConv3D, Conv3D, BatchNorm, ReLU


nn = _NN()
