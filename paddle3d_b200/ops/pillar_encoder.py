"""SURVEY.md §8a-5 / §8f-2 (tests/test_gpu_voxelize.py): PillarFeatureNet (models/voxel_encoders/pillar_encoder.py:
115-210) with one PFNLayer (PointPillars) or two (CenterPoint-pillars) as one launch over the `hard_voxelize` outputs."""
import numpy as np
import torch

from .._lib import check, host_floats, lib
from .._mem import ptr, require_cuda, stream

WIDE_FROM = 65  # points per pillar from which pillar_feature_net2 launches p3d_pillar_feature_net2_wide


def fold_bn(bn_gamma, bn_beta, bn_mean, bn_var, bn_eps, device):
    """BatchNorm1D(eval) as (scale, shift) device tensors, folded on the host in fp64: do this once per model."""
    s = np.asarray(bn_gamma, np.float64) / np.sqrt(np.asarray(bn_var, np.float64) + bn_eps)
    t = np.asarray(bn_beta, np.float64) - np.asarray(bn_mean, np.float64) * s
    return torch.from_numpy(s.astype(np.float32)).to(device), torch.from_numpy(t.astype(np.float32)).to(device)


def pillar_feature_net(voxels, num_points_per_voxel, coors, weight, bn_gamma, bn_beta, bn_mean, bn_var, bn_eps,
                       voxel_size, point_cloud_range, num_voxels=None, folded=None):
    """voxels [n, M, F], counts [n], coors [n, 4] (b, z, y, x) int32, weight [F + 5, C] -> [n, C] pillar features.
    folded: (scale, shift) from fold_bn - pass it to keep host->device copies out of the per-frame path (CUDA graphs)."""
    voxels = require_cuda(voxels, "voxels", torch.float32)
    npv = require_cuda(num_points_per_voxel, "num_points_per_voxel", torch.int32)
    coors = require_cuda(coors, "coors", torch.int32)
    weight = require_cuda(weight, "weight", torch.float32)
    n, m, f = voxels.shape
    c = weight.shape[1]
    if weight.shape[0] != f + 5:
        raise ValueError("weight must be [F + 5, C]")
    dev = voxels.device
    scale, shift = folded if folded is not None else fold_bn(bn_gamma, bn_beta, bn_mean, bn_var, bn_eps, dev)
    out = torch.zeros((n, c), dtype=torch.float32, device=dev)
    nump = ptr(require_cuda(num_voxels, "num_voxels", torch.int32)) if num_voxels is not None else ptr(None)
    check(lib().p3d_pillar_feature_net(ptr(voxels), ptr(npv), ptr(coors), nump, n, m, f, c, ptr(weight), ptr(scale),
                                       ptr(shift), host_floats(voxel_size), host_floats(point_cloud_range), ptr(out),
                                       stream(dev)), "pillar_feature_net")
    return out


def pillar_feature_net2(voxels, num_points_per_voxel, coors, layers, voxel_size, point_cloud_range, num_voxels=None,
                        folded=None):
    """PillarFeatureNet with two PFNLayers (CenterPoint-pillars, feat_channels [64, 64]) as one launch.  layers: two dicts
    of weight / gamma / beta / mean / var / eps, weight [F + 5, mid] then [2 mid, out] on the device.  folded: the two
    (scale, shift) pairs of fold_bn, to keep host->device copies out of the per-frame path.  Returns [n, out].  Up to 64
    points per pillar run on p3d_pillar_feature_net2, 65 to 128 on p3d_pillar_feature_net2_wide (same arithmetic, more
    shared memory per pillar)."""
    voxels = require_cuda(voxels, "voxels", torch.float32)
    npv = require_cuda(num_points_per_voxel, "num_points_per_voxel", torch.int32)
    coors = require_cuda(coors, "coors", torch.int32)
    w1 = require_cuda(layers[0]["weight"], "layers[0].weight", torch.float32)
    w2 = require_cuda(layers[1]["weight"], "layers[1].weight", torch.float32)
    n, m, f = voxels.shape
    mid, c = w1.shape[1], w2.shape[1]
    if w1.shape[0] != f + 5 or w2.shape[0] != 2 * mid:
        raise ValueError("weights must be [F + 5, mid] and [2 mid, out]")
    dev = voxels.device
    if folded is None:
        folded = [fold_bn(l["gamma"], l["beta"], l["mean"], l["var"], l["eps"], dev) for l in layers]
    (s1, t1), (s2, t2) = folded
    out = torch.zeros((n, c), dtype=torch.float32, device=dev)
    nump = ptr(require_cuda(num_voxels, "num_voxels", torch.int32)) if num_voxels is not None else ptr(None)
    fn = lib().p3d_pillar_feature_net2 if m < WIDE_FROM else lib().p3d_pillar_feature_net2_wide
    check(fn(ptr(voxels), ptr(npv), ptr(coors), nump, n, m, f, mid, ptr(w1), ptr(s1), ptr(t1), c, ptr(w2), ptr(s2), ptr(t2),
             host_floats(voxel_size), host_floats(point_cloud_range), ptr(out), stream(dev)), "pillar_feature_net2")
    return out


def hard_vfe(voxels, num_points_per_voxel, coors, layers, voxel_size, point_cloud_range, num_voxels=None, folded=None,
             out=None):
    """mmdet3d HardVFE (feat_channels [mid, out], with_cluster_center, with_voxel_center, no distance) as one launch
    (p3d_hard_vfe): the decoration adds xyz minus the voxel centre, z included, and the first layer is not halved.
    layers: two dicts of weight / gamma / beta / mean / var / eps, weight [F + 6, mid] then [2 mid, out] on the device.
    voxel_size: 3 values, point_cloud_range: 6.  folded: the two (scale, shift) pairs of fold_bn.  out: an existing
    [n, out] fp32 buffer (a captured frame keeps its address; rows past num_voxels are left as they are), default a new
    zero-filled one.  Returns the [n, out] features."""
    voxels = require_cuda(voxels, "voxels", torch.float32)
    npv = require_cuda(num_points_per_voxel, "num_points_per_voxel", torch.int32)
    coors = require_cuda(coors, "coors", torch.int32)
    w1 = require_cuda(layers[0]["weight"], "layers[0].weight", torch.float32)
    w2 = require_cuda(layers[1]["weight"], "layers[1].weight", torch.float32)
    n, m, f = voxels.shape
    mid, c = w1.shape[1], w2.shape[1]
    if w1.shape[0] != f + 6 or w2.shape[0] != 2 * mid:
        raise ValueError("weights must be [F + 6, mid] and [2 mid, out]")
    if len(voxel_size) != 3 or len(point_cloud_range) != 6:
        raise ValueError("voxel_size needs 3 values and point_cloud_range 6")
    dev = voxels.device
    if folded is None:
        folded = [fold_bn(l["gamma"], l["beta"], l["mean"], l["var"], l["eps"], dev) for l in layers]
    (s1, t1), (s2, t2) = folded
    if out is None:
        out = torch.zeros((n, c), dtype=torch.float32, device=dev)
    elif tuple(out.shape) != (n, c) or out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous():
        raise ValueError("out must be a contiguous [n, out] fp32 device tensor")
    nump = ptr(require_cuda(num_voxels, "num_voxels", torch.int32)) if num_voxels is not None else ptr(None)
    check(lib().p3d_hard_vfe(ptr(voxels), ptr(npv), ptr(coors), nump, n, m, f, mid, ptr(w1), ptr(s1), ptr(t1), c, ptr(w2),
                             ptr(s2), ptr(t2), host_floats(voxel_size), host_floats(point_cloud_range), ptr(out),
                             stream(dev)), "hard_vfe")
    return out
