"""Multi-sweep merge on the device (csrc/sweep_merge.cu): LoadPointCloud.__call__ (paddle3d/transforms/reader.py:116-167)
as one kernel pass over raw sweep rows already on the GPU.  The reference has no op for it (it is a data transform);
`io.merge_sweeps` is the host restatement every result here is compared against.  The same pass with the KITTI camera
frustum cull (merge_frustum_into / frustum_cull_device) has `kitti.remove_camera_invisible` as its host restatement."""
import numpy as np
import torch

from .._lib import check, host_ints, lib
from .._mem import ptr, require_cuda, stream, workspace

# struct p3d_sweep_desc (include/p3d_b200.h), one entry per sweep of a frame: key first, then merge order
DESC_DTYPE = np.dtype([("slot", "<i4"), ("rows", "<i4"), ("has_transform", "<i4"), ("time_lag", "<f4"),
                       ("ref_from_curr", "<f8", (12,))])
assert DESC_DTYPE.itemsize == 112

OVERFLOW, BAD_ENTRY = 1, 2  # bits of the status word


def columns(use_dim, raw_dim):
    """Selected raw columns (reader.py:123-126, 139-140): None = all of them, int k = the first k, or a list."""
    if use_dim is None:
        return list(range(raw_dim))
    cols = list(range(int(use_dim))) if isinstance(use_dim, (int, np.integer)) else [int(c) for c in use_dim]
    if not cols:  # the reference's key frame then keeps no column while its sweeps keep all: no merged cloud exists
        raise ValueError("use_dim selects no column")
    if min(cols) < 0 or max(cols) >= raw_dim or len(cols) < 3:
        raise ValueError("use_dim %r: need >= 3 columns in [0, %d)" % (use_dim, raw_dim))
    return cols


def set_entry(entry, slot, rows, ref_from_curr=None, time_lag=0.0):
    """Fill one descriptor entry; ref_from_curr: 4x4 or 3x4 (any float dtype, used in float64) or None."""
    entry["slot"], entry["rows"] = int(slot), int(rows)
    entry["time_lag"] = np.float32(time_lag)
    if ref_from_curr is None:
        entry["has_transform"] = 0
        entry["ref_from_curr"] = 0.0
    else:
        m = np.asarray(ref_from_curr, np.float64)
        if m.shape not in ((4, 4), (3, 4)):
            raise ValueError("ref_from_curr must be 4x4 or 3x4, got %s" % (m.shape,))
        entry["has_transform"] = 1
        entry["ref_from_curr"] = m[:3].reshape(12)


def merge_into(raw, desc_dev, num_entries, cols, use_time_lag, sweep_remove_radius, out, n_out, status):
    """Enqueue the merge on the current stream (all arguments on the device; the CUDA-graph form).
    raw [slots, slot_cap, raw_dim] fp32; desc_dev: uint8 [num_entries * 112]; out [cap, F] fp32; n_out / status [1] int32."""
    slots, slot_cap, raw_dim = raw.shape
    cap, F = out.shape
    if F != len(cols) + bool(use_time_lag) or desc_dev.numel() < num_entries * DESC_DTYPE.itemsize:
        raise ValueError("merge_sweeps: output has %d columns, descriptor %d bytes" % (F, desc_dev.numel()))
    L = lib()
    ws = workspace(L.p3d_merge_sweeps_workspace_bytes(num_entries, slot_cap), raw.device, "sweep_merge")
    check(L.p3d_merge_sweeps(ptr(raw), slots, slot_cap, raw_dim, ptr(desc_dev), num_entries, host_ints(cols), len(cols),
                             int(bool(use_time_lag)), float(np.float32(sweep_remove_radius)), ptr(out), cap, ptr(n_out),
                             ptr(status), ptr(ws), ws.numel(), stream(raw.device)), "merge_sweeps")


def merge_frustum_into(raw, desc_dev, planes_dev, cols, out, n_out, status, num_entries=1):
    """merge_into of the one entry of desc_dev with the camera frustum cull (p3d_merge_sweeps_frustum): rows outside the
    six planes of planes_dev [6, 4] fp64 (device; kitti.frustum_planes) are dropped, order kept.  No time lag, no
    removal square.  num_entries != 1 is refused by the library (P3DError)."""
    slots, slot_cap, raw_dim = raw.shape
    cap, F = out.shape
    if F != len(cols) or desc_dev.numel() < num_entries * DESC_DTYPE.itemsize:
        raise ValueError("merge_sweeps_frustum: output has %d columns, descriptor %d bytes" % (F, desc_dev.numel()))
    if planes_dev.dtype != torch.float64 or planes_dev.numel() != 24 or not planes_dev.is_contiguous():
        raise ValueError("merge_sweeps_frustum: planes must be a contiguous [6, 4] float64 device tensor")
    L = lib()
    ws = workspace(L.p3d_merge_sweeps_workspace_bytes(num_entries, slot_cap), raw.device, "sweep_merge")
    check(L.p3d_merge_sweeps_frustum(ptr(raw), slots, slot_cap, raw_dim, ptr(desc_dev), num_entries, host_ints(cols),
                                     len(cols), 0, 0.0, ptr(out), cap, ptr(n_out), ptr(status), ptr(ws), ws.numel(),
                                     stream(raw.device), ptr(planes_dev)), "merge_sweeps_frustum")


def frustum_cull_device(cloud, planes, cap=None, use_dim=None, device="cuda"):
    """kitti.remove_camera_invisible on the GPU: cloud [n, raw_dim] fp32, planes [6, 4] (kitti.frustum_planes).  Returns
    (points [cap, F] fp32 on the device, NaN rows from n_out on, n_out [1] int32, status [1] int32: OVERFLOW when more than
    cap rows were kept).  cap defaults to n."""
    cloud = np.ascontiguousarray(cloud, np.float32)
    if cloud.ndim != 2:
        raise ValueError("cloud must be [n, raw_dim]")
    raw_dim = cloud.shape[1]
    cols = columns(use_dim, raw_dim)
    slot_cap = max(4, -(-len(cloud) // 4) * 4)
    host = np.zeros((1, slot_cap, raw_dim), np.float32)
    host[0, :len(cloud)] = cloud
    desc = np.zeros(1, DESC_DTYPE)
    set_entry(desc[0], 0, len(cloud))
    dev = torch.device(device)
    cap = len(cloud) if cap is None else int(cap)
    out = torch.empty((cap, len(cols)), dtype=torch.float32, device=dev)
    n_out = torch.empty((1,), dtype=torch.int32, device=dev)
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    raw = torch.from_numpy(host).to(dev)
    planes_dev = torch.from_numpy(np.ascontiguousarray(planes, np.float64).reshape(6, 4)).to(dev)
    merge_frustum_into(raw, torch.from_numpy(desc.view(np.uint8)).to(dev), planes_dev, cols, out, n_out, status)
    return out, n_out, status


def merge_sweeps_device(key, sweeps=(), use_dim=None, use_time_lag=False, sweep_remove_radius=1.0, order=None, cap=None,
                        device="cuda"):
    """Same arguments as io.merge_sweeps (key [n, raw_dim] fp32, sweeps [(cloud, ref_from_curr | None, time_lag)]),
    computed on the GPU.  Returns (points [cap, F] fp32 on the device, NaN rows from n_out on, n_out [1] int32,
    status [1] int32: OVERFLOW when the merge did not fit in cap, rows beyond it dropped).  cap defaults to the rows of
    the key plus every sweep."""
    key = np.ascontiguousarray(key, np.float32)
    raw_dim = key.shape[1]
    cols = columns(use_dim, raw_dim)
    idx = list(range(len(sweeps))) if order is None else [int(i) for i in order]
    if sorted(idx) != list(range(len(sweeps))):
        raise ValueError("order must be a permutation of the sweep indices")
    clouds = [key] + [np.ascontiguousarray(sweeps[i][0], np.float32) for i in idx]
    if any(c.ndim != 2 or c.shape[1] != raw_dim for c in clouds):
        raise ValueError("every cloud must be [n, %d]" % raw_dim)
    slot_cap = max(4, -(-max(len(c) for c in clouds) // 4) * 4)
    host = np.zeros((len(clouds), slot_cap, raw_dim), np.float32)
    desc = np.zeros(len(clouds), DESC_DTYPE)
    for e, c in enumerate(clouds):
        host[e, :len(c)] = c
        m, lag = (None, 0.0) if e == 0 else (sweeps[idx[e - 1]][1], sweeps[idx[e - 1]][2])
        set_entry(desc[e], e, len(c), m, lag)
    dev = torch.device(device)
    cap = sum(len(c) for c in clouds) if cap is None else int(cap)
    out = torch.empty((cap, len(cols) + bool(use_time_lag)), dtype=torch.float32, device=dev)
    n_out = torch.empty((1,), dtype=torch.int32, device=dev)
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    raw = torch.from_numpy(host).to(dev)
    desc_dev = torch.from_numpy(desc.view(np.uint8)).to(dev)
    require_cuda(raw, "raw", torch.float32)
    merge_into(raw, desc_dev, len(clouds), cols, use_time_lag, sweep_remove_radius, out, n_out, status)
    return out, n_out, status
