"""Drop-in mirror of `paddle3d.ops` for the point-cloud-to-BEV hot path.

Module and function names, argument order and meaning follow the reference's generated custom-op
modules (paddle3d/ops/__init__.py:27-104 lists them; SURVEY.md §8b lists the call sites):

    from paddle3d_b200.ops import voxelize, iou3d_nms, centerpoint_postprocess, bev_pool_v2, bev_pool_v2_backward

plus the two layer-level entry points whose arithmetic lives inside PaddlePaddle in the reference:
`pillar_scatter` (paddle.scatter in PointPillarsScatter) and `sparse_nn` (paddle.sparse.nn), and
`bevdet_postprocess`, BEVDet's own box decode (scale-NMS / circle NMS), which the reference runs in Python.
Tensors are torch CUDA tensors (Paddle is not installable in this image; under Paddle the same C ABI
is bound by paddle_ext/*.cc, see INTEGRATION.md).
"""
from . import (bev_pool_v2, bev_pool_v2_backward, bevdet_postprocess, centerpoint_postprocess, iou3d_nms, pillar_scatter,  # noqa: F401
               sparse_nn, voxelize)

custom_ops = {  # same keys as paddle3d/ops/__init__.py:27-104 for the ops on this path
    "voxelize": voxelize,
    "iou3d_nms": iou3d_nms,
    "centerpoint_postprocess": centerpoint_postprocess,
    "bev_pool_v2": bev_pool_v2,
    "bev_pool_v2_backward": bev_pool_v2_backward,
}
