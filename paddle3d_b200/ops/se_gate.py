"""BEVFusion's SE_Block (x * sigmoid(Conv1x1_bias(mean_hw(x)))) in place on a pixel H16 image — op `p3d_se_gate_h16`
(include/p3d_b200.h states its rounding; PARITY UNPINNED: recalled from ADLab's BEVFusion)."""
import torch

from .._lib import check, lib
from .._mem import ptr, require_cuda, stream, workspace
from .dense_conv import _status


def se_gate_h16(x_h16, shape, weight, bias, gate=None, status=None):
    """x_h16 [B*H*W, 2*C] float16 pixel H16 rows, shape = (B, H, W, C), scaled in place.  weight [C, C] (the 1x1 conv's
    [out, in]) and bias [C] fp32 on the device.  gate: an fp32 [B, C] device buffer for the gate (None: a new one).
    status: the int32 word bit 0 is OR-ed into (None: the device's fp16-pair status word).  Returns the gate."""
    x_h16 = require_cuda(x_h16, "x_h16", torch.float16)
    weight = require_cuda(weight, "weight", torch.float32)
    bias = require_cuda(bias, "bias", torch.float32)
    b, h, w, c = [int(v) for v in shape]
    if x_h16.numel() != b * h * w * 2 * c:
        raise ValueError("x_h16 must hold B*H*W rows of 2*C halves")
    if tuple(weight.shape) not in ((c, c), (c, c, 1, 1)) or tuple(bias.shape) != (c,):
        raise ValueError("weight must be [C, C] and bias [C]")
    dev = x_h16.device
    if gate is None:
        gate = torch.empty((b, c), dtype=torch.float32, device=dev)
    status = _status(dev) if status is None else status
    L = lib()
    ws = workspace(L.p3d_se_gate_workspace_bytes(b, h, w, c), dev, "se_gate")
    check(L.p3d_se_gate_h16(ptr(x_h16), b, h, w, c, ptr(weight), ptr(bias), ptr(gate), ptr(status), ptr(ws), ws.numel(),
                            stream(dev)), "se_gate_h16")
    return gate
