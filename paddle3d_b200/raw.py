"""Torch-free front end: the C ABI driven with nothing but ctypes + libcudart + numpy.

The library itself never depended on torch (include/p3d_b200.h takes plain pointers, sizes and a stream); the Python
mirror under `paddle3d_b200/ops` uses torch as its allocator / stream provider, the role Paddle's allocator plays under
`paddle_ext/`.  This module is the same boundary WITHOUT torch (BASELINE north_star: "no PyTorch"): a minimal
device-buffer class over `cudaMalloc`, a stream, and numpy-in / numpy-out versions of the reference ops whose whole
signature is arrays (`hard_voxelize`, `boxes_iou_bev`, `nms_gpu`).  `import paddle3d_b200.raw` does not import torch
(`tests/test_gpu_raw.py` checks that in a fresh interpreter).  There is no CPU fallback here either.
"""
import ctypes as C
import ctypes.util

import numpy as np

from ._lib import P3DError, check, lib

_H2D, _D2H = 1, 2
_rt = None


def cudart():
    """libcudart via ctypes (the runtime libp3d_b200.so itself links)."""
    global _rt
    if _rt is None:
        last = None
        for name in ("libcudart.so.12", ctypes.util.find_library("cudart"), "/usr/local/cuda/lib64/libcudart.so"):
            if not name:
                continue
            try:
                _rt = C.CDLL(name)
                break
            except OSError as e:  # try the next spelling
                last = e
        if _rt is None:
            raise P3DError("libcudart not found (%s): paddle3d_b200.raw needs the CUDA runtime" % last)
        _rt.cudaMalloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
        _rt.cudaFree.argtypes = [C.c_void_p]
        _rt.cudaMemcpyAsync.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
        _rt.cudaMemcpy2DAsync.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                          C.c_int, C.c_void_p]
        _rt.cudaMemsetAsync.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_void_p]
        _rt.cudaStreamCreate.argtypes = [C.POINTER(C.c_void_p)]
        _rt.cudaStreamDestroy.argtypes = [C.c_void_p]
        _rt.cudaStreamSynchronize.argtypes = [C.c_void_p]
        _rt.cudaSetDevice.argtypes = [C.c_int]
        _rt.cudaGetErrorString.restype = C.c_char_p
        _rt.cudaGetErrorString.argtypes = [C.c_int]
    return _rt


def _ok(rc, what):
    if rc != 0:
        raise P3DError("%s: %s (cudaError %d)" % (what, cudart().cudaGetErrorString(rc).decode(), rc))


def set_device(index):
    _ok(cudart().cudaSetDevice(int(index)), "cudaSetDevice")


class Stream:
    def __init__(self):
        self.handle = C.c_void_p()
        _ok(cudart().cudaStreamCreate(C.byref(self.handle)), "cudaStreamCreate")

    def synchronize(self):
        _ok(cudart().cudaStreamSynchronize(self.handle), "cudaStreamSynchronize")

    def __del__(self):
        if getattr(self, "handle", None) and _rt is not None:
            _rt.cudaStreamDestroy(self.handle)
            self.handle = None


class DeviceBuffer:
    """`nbytes` of device memory (256-byte aligned by cudaMalloc); freed with the object."""

    def __init__(self, nbytes, zero=False, stream=None):
        self.nbytes = max(int(nbytes), 16)
        self.ptr = C.c_void_p()
        _ok(cudart().cudaMalloc(C.byref(self.ptr), self.nbytes), "cudaMalloc(%d)" % self.nbytes)
        if zero:
            _ok(cudart().cudaMemsetAsync(self.ptr, 0, self.nbytes, stream.handle if stream else None), "cudaMemsetAsync")

    @classmethod
    def from_host(cls, array, stream=None):
        a = np.ascontiguousarray(array)
        b = cls(a.nbytes)
        b.upload(a, stream)
        return b

    def upload(self, array, stream=None):
        a = np.ascontiguousarray(array)
        if a.nbytes > self.nbytes:
            raise P3DError("upload of %d bytes into a %d-byte buffer" % (a.nbytes, self.nbytes))
        _ok(cudart().cudaMemcpyAsync(self.ptr, a.ctypes.data_as(C.c_void_p), a.nbytes, _H2D, stream.handle if stream else None),
            "cudaMemcpyAsync H2D")
        if stream is None:
            _ok(cudart().cudaStreamSynchronize(None), "cudaStreamSynchronize")  # pageable source: finish before `a` can go away
        else:
            stream.synchronize()

    def download(self, shape, dtype, stream=None):
        out = np.empty(shape, dtype)
        if out.nbytes > self.nbytes:
            raise P3DError("download of %d bytes from a %d-byte buffer" % (out.nbytes, self.nbytes))
        _ok(cudart().cudaMemcpyAsync(out.ctypes.data_as(C.c_void_p), self.ptr, out.nbytes, _D2H, stream.handle if stream else None),
            "cudaMemcpyAsync D2H")
        if stream is None:
            _ok(cudart().cudaStreamSynchronize(None), "cudaStreamSynchronize")
        else:
            stream.synchronize()
        return out

    def __del__(self):
        if getattr(self, "ptr", None) and _rt is not None:
            _rt.cudaFree(self.ptr)
            self.ptr = None


def _floats(v):
    return (C.c_float * len(v))(*[float(x) for x in v])


def hard_voxelize(points, voxel_size, point_cloud_range, max_num_points_in_voxel, max_voxels, stream=None):
    """paddle3d.ops.voxelize.hard_voxelize (voxelize_op.cc:183-191) on a host array: numpy in, numpy out
    (voxels [V,P,F] fp32, coords [V,3] int32 (z,y,x), num_points_per_voxel [V] int32, num_voxels [1] int32)."""
    pts = np.ascontiguousarray(points, np.float32)
    if pts.ndim != 2 or pts.shape[1] < 3:
        raise ValueError("points must be [N, >=3]")
    n, f = pts.shape
    P, V = int(max_num_points_in_voxel), int(max_voxels)
    st = stream or Stream()
    L = lib()
    d_pts = DeviceBuffer.from_host(pts, st)
    d_vox, d_coords = DeviceBuffer(V * P * f * 4), DeviceBuffer(V * 3 * 4)
    d_npv, d_nv = DeviceBuffer(V * 4), DeviceBuffer(4)
    ws_bytes = L.p3d_hard_voxelize_workspace_bytes(n, P, V)
    d_ws = DeviceBuffer(ws_bytes)
    check(L.p3d_hard_voxelize(d_pts.ptr, n, f, _floats(voxel_size), _floats(point_cloud_range), P, V, d_vox.ptr, d_coords.ptr,
                              d_npv.ptr, d_nv.ptr, d_ws.ptr, ws_bytes, st.handle), "hard_voxelize")
    return (d_vox.download((V, P, f), np.float32, st), d_coords.download((V, 3), np.int32, st),
            d_npv.download((V,), np.int32, st), d_nv.download((1,), np.int32, st))


def boxes_iou_bev(boxes_a, boxes_b, stream=None):
    """iou3d_nms.boxes_iou_bev_gpu (iou3d_nms.cpp:62-84): [M, 7] x [N, 7] -> [M, N] fp32 rotated BEV IoU."""
    a, b = np.ascontiguousarray(boxes_a, np.float32), np.ascontiguousarray(boxes_b, np.float32)
    st = stream or Stream()
    d_a, d_b = DeviceBuffer.from_host(a, st), DeviceBuffer.from_host(b, st)
    d_o = DeviceBuffer(a.shape[0] * b.shape[0] * 4)
    check(lib().p3d_boxes_iou_bev(d_a.ptr, a.shape[0], d_b.ptr, b.shape[0], d_o.ptr, st.handle), "boxes_iou_bev")
    return d_o.download((a.shape[0], b.shape[0]), np.float32, st)


def nms_gpu(boxes, nms_overlap_thresh, normal=False, stream=None):
    """iou3d_nms.nms_gpu / nms_normal_gpu (iou3d_nms.cpp:86-204): boxes sorted by score -> (keep int32 [N], num_to_keep)."""
    bx = np.ascontiguousarray(boxes, np.float32)
    n = bx.shape[0]
    st = stream or Stream()
    L = lib()
    d_b, d_keep, d_num = DeviceBuffer.from_host(bx, st), DeviceBuffer(max(n, 1) * 4), DeviceBuffer(4)
    ws_bytes = L.p3d_nms_workspace_bytes(n)
    d_ws = DeviceBuffer(ws_bytes)
    check(L.p3d_nms(d_b.ptr, n, float(nms_overlap_thresh), int(bool(normal)), d_keep.ptr, d_num.ptr, d_ws.ptr, ws_bytes,
                    st.handle), "nms")
    return d_keep.download((n,), np.int32, st), int(d_num.download((1,), np.int32, st)[0])
