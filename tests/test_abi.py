"""CPU suite: the C-ABI library loads and exports every symbol include/p3d_b200.h declares;
the host mirror refuses to run without CUDA tensors (no fallback).  No compute calls."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def _declared():
    src = open(os.path.join(ROOT, "include", "p3d_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(p3d_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), "missing export %s" % n
        assert n in _lib.SIGNATURES, "no ctypes signature for %s" % n
    assert lib.p3d_abi_version() == 1


def test_status_strings_and_size_queries():
    from paddle3d_b200 import _lib
    L = _lib.lib()
    assert L.p3d_status_string(0) == b"ok"
    assert b"workspace" in L.p3d_status_string(-2)
    assert L.p3d_hard_voxelize_workspace_bytes(300000, 10, 160000) > 8 * 2 ** 20
    assert L.p3d_hard_voxelize_workspace_bytes(-1, 10, 10) == 0
    assert L.p3d_nms_workspace_bytes(1000) >= 1000 * 16 * 8
    assert L.p3d_scatter_dense_workspace_bytes(1, 1, 496, 432) >= 496 * 432 * 4
    assert L.p3d_centerpoint_postprocess_workspace_bytes(6, 180, 180, 1000, 83) > 0
    assert L.p3d_sparse_rulebook_workspace_bytes(160000, 640000) > 0
    # the scratch-workspace rulebook calls hold one table per index set (512-row floor each)
    for n_in, n_out in ((160000, 640000), (1000, 0), (0, 0)):
        want = L.p3d_sparse_table_bytes(n_in) + L.p3d_sparse_table_bytes(n_out)
        assert L.p3d_sparse_rulebook_workspace_bytes(n_in, n_out) == want
    # capacities whose hash table (2x rows, power of two) would not fit 2^31 entries are refused, not looped on (ADVICE r1)
    assert L.p3d_hard_voxelize_workspace_bytes(2 ** 31, 10, 10) == 0
    assert L.p3d_sparse_table_bytes(2 ** 31 + 5) == 0
    assert L.p3d_sparse_rulebook_workspace_bytes(2 ** 31, 16) == 0
    # the narrow-layer warp-MMA kernel: supported shapes only
    assert L.p3d_sparse_conv_wm_packed_weight_bytes(27, 16, 16) == 27 * 1024
    assert L.p3d_sparse_conv_wm_packed_weight_bytes(27, 32, 32) == 27 * 4 * 1024
    assert L.p3d_sparse_conv_wm_packed_weight_bytes(27, 64, 64) == 0
    assert L.p3d_sparse_conv_wm_workspace_bytes(1000, 16) > 0


def test_host_mirror_rejects_cpu_tensors():
    import torch
    from paddle3d_b200 import _lib
    from paddle3d_b200.ops import iou3d_nms, voxelize
    with pytest.raises(_lib.P3DError):
        voxelize.hard_voxelize(torch.zeros(10, 4), [0.16, 0.16, 4], [0, -39.68, -3, 69.12, 39.68, 1], 32, 100)
    with pytest.raises(_lib.P3DError):
        iou3d_nms.boxes_iou_bev_cpu(torch.zeros(2, 7), torch.zeros(2, 7))


def test_invalid_arguments_return_status_codes():
    from paddle3d_b200 import _lib
    L = _lib.lib()
    vs = _lib.host_floats([0.1, 0.1, 0.1])
    pcr = _lib.host_floats([0, 0, 0, 1, 1, 1])
    # null outputs -> invalid argument, before any CUDA call
    rc = L.p3d_hard_voxelize(None, 0, 4, vs, pcr, 4, 16, None, None, None, None, None, 0, None)
    assert rc == -1
    # grid too large for 31-bit cell ids -> unsupported
    big = _lib.host_floats([0, 0, 0, 1e5, 1e5, 1e3])
    tiny = _lib.host_floats([0.01, 0.01, 0.01])
    rc = L.p3d_hard_voxelize(None, 0, 4, tiny, big, 4, 16, None, None, None, None, None, 0, None)
    assert rc == -4
    assert L.p3d_nms(None, -1, 0.5, 0, None, None, None, 0, None) == -1
    # 17 tasks is more than the postprocess batches: unsupported, decided before any pointer is read; 0 tasks is invalid
    for tasks, rc in ((17, -4), (0, -1)):
        assert L.p3d_centerpoint_postprocess(tasks, *[None] * 7, 180, 180, *[None] * 4, 8, 0.1, 0.2, 1000, 83, 1,
                                             *[None] * 5, 0, None) == rc


def test_conv_entry_points_reject_invalid_arguments():
    """Host-side validation of the sparse / dense conv entry points: every call below must be rejected before any
    CUDA call is made (no GPU here)."""
    import ctypes as C
    from paddle3d_b200 import _lib
    L = _lib.lib()
    p = C.c_void_p(256)  # a non-null, 16-byte aligned dummy address: the checks below fail before it is touched
    odd = C.c_void_p(260)  # misaligned
    # sparse split-row conv: K out of range, missing outputs, misaligned rows, unsupported channel counts
    assert L.p3d_sparse_conv_gather_gemm_split_ws(p, p, None, 128, 0, 32, 32, p, None, None, None, 0, p, None, None, 0, None) == -1
    assert L.p3d_sparse_conv_gather_gemm_split_ws(p, p, None, 128, 27, 32, 32, p, None, None, None, 0, None, None, None, 0, None) == -1
    assert L.p3d_sparse_conv_gather_gemm_split_ws(odd, p, None, 128, 27, 32, 32, p, None, None, None, 0, p, None, None, 0, None) == -1
    assert L.p3d_sparse_conv_gather_gemm_split_ws(p, p, None, 128, 27, 48, 48, p, None, None, None, 0, p, None, None, 0, None) == -4
    # sparse fp32-row conv on the same kernel: K out of range, misaligned rows, unsupported channel counts
    assert L.p3d_sparse_conv_gather_gemm_tf32x3_ws(p, p, None, 128, 0, 32, 32, p, None, None, None, 0, p, None, 0, None) == -1
    assert L.p3d_sparse_conv_gather_gemm_tf32x3_ws(odd, p, None, 128, 27, 32, 32, p, None, None, None, 0, p, None, 0, None) == -1
    assert L.p3d_sparse_conv_gather_gemm_tf32x3_ws(p, p, None, 128, 27, 48, 48, p, None, None, None, 0, p, None, 0, None) == -4
    assert L.p3d_sparse_conv_packed_weight_bytes(27, 5, 16) == 0 and L.p3d_sparse_conv_packed_weight_bytes(27, 16, 16) > 0
    assert L.p3d_rows_convert_layout(p, 2, None, 16, 16, p, None) == -1
    # narrow-layer warp-MMA conv: unsupported shape, missing output, misaligned neighbour map, missing / short workspace
    wm = L.p3d_sparse_conv_wm
    assert wm(p, p, None, 128, 27, 64, 64, p, None, None, None, 0, p, None, p, 1 << 30, None, None) == -4
    assert wm(p, p, None, 128, 27, 16, 16, p, None, None, None, 0, None, None, p, 1 << 30, None, None) == -1
    assert wm(p, odd, None, 128, 27, 16, 16, p, None, None, None, 0, p, None, p, 1 << 30, None, None) == -1
    assert wm(p, p, None, 128, 27, 16, 16, p, None, None, None, 0, p, None, None, 0, None, None) == -2
    assert wm(p, p, None, 128, 27, 16, 16, p, None, None, None, 0, p, None, p, 16, None, None) == -2
    assert wm(p, p, None, 0, 27, 16, 16, p, None, None, None, 0, p, None, None, 0, None, None) == 0  # empty input: nothing to do
    # fp16-pair wgmma conv: K out of range, missing output, misaligned rows, unsupported channel counts
    f16 = L.p3d_sparse_conv_f16
    assert f16(p, p, None, 128, 0, 32, 32, p, None, None, None, 0, p, None, None, 0, 4, None, None) == -1
    assert f16(p, p, None, 128, 33, 32, 32, p, None, None, None, 0, p, None, None, 0, 4, None, None) == -1
    assert f16(p, p, None, 128, 27, 32, 32, p, None, None, None, 0, None, None, None, 0, 4, None, None) == -1
    assert f16(odd, p, None, 128, 27, 32, 32, p, None, None, None, 0, p, None, None, 0, 4, None, None) == -1
    assert f16(p, p, None, 128, 27, 48, 48, p, None, None, None, 0, p, None, None, 0, 4, None, None) == -4
    assert f16(p, p, None, 128, 27, 32, 48, p, None, None, None, 0, p, None, None, 0, 4, None, None) == -4
    # dense conv: channel counts, N tile, transposed-conv geometry, split-row output columns
    ok = dict(B=1, H=8, W=8)
    assert L.p3d_dense_conv2d_split(p, 1, 8, 8, 48, p, 64, 64, 3, 3, 1, 1, 1, None, None, 0, p, 64, 0, None, None) == -4
    assert L.p3d_dense_conv2d_split(p, 1, 8, 8, 64, p, 64, 32, 3, 3, 1, 1, 1, None, None, 0, p, 64, 0, None, None) == -4
    assert L.p3d_dense_conv2d_split(p, 1, 8, 8, 64, p, 64, 64, 3, 3, 2, 1, 2, None, None, 0, p, 64, 0, None, None) == -4
    assert L.p3d_dense_conv2d_split(p, 1, 8, 8, 64, p, 64, 64, 3, 3, 1, 1, 1, None, None, 0, None, 64, 0, None, None) == -1
    assert L.p3d_dense_conv2d_split(p, 1, 8, 8, 64, p, 64, 64, 3, 3, 1, 1, 1, None, None, 0, p, 96, 64, None, None) == -1
    assert L.p3d_dense_conv2d_packed_weight_bytes(9, 64, 70, 16) == 5 * 9 * 64 * 32 * 4
    assert L.p3d_dense_conv2d_packed_weight_bytes(9, 48, 64, 64) == 0
    # fp16-pair dense conv: mode 0 (auto) or 1 (per-tap loads) only
    assert L.p3d_dense_conv2d_f16(p, 1, 8, 8, 64, p, 64, 64, 3, 3, 1, 1, 1, None, None, 0, p, 64, 0, None, 2, 0, None, None) == -1
    # grouped head output conv and the pillar encoder
    assert L.p3d_head_final_conv(p, 1, 8, 8, 128, 64, 3, p, p, p, p, 8, p, None) == -1     # 3 * 64 > 128 channels
    assert L.p3d_head_out_conv_f16(p, 1, 8, 8, 352, 352, 1, p, p, None, p, p, 3, p, None) == -4  # < 2 activation slots
    assert L.p3d_pillar_feature_net(p, p, p, None, 10, 100, 4, 64, p, p, p, p, p, p, None) == -4  # > 64 points / pillar
    assert L.p3d_pillar_feature_net(p, p, p, None, 10, 32, 4, 64, None, p, p, p, p, p, None) == -1


def test_paddle_glue_compiles():
    """paddle_ext/p3d_paddle_ops.cc (the PD_BUILD_OP registrations that bind the C ABI under PaddlePaddle) must at
    least compile against the stub extension header: PaddlePaddle itself is not installable here."""
    import subprocess
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "oracle", "stub"), "-I",
                        os.path.join(ROOT, "include"), os.path.join(ROOT, "paddle_ext", "p3d_paddle_ops.cc")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    src = open(os.path.join(ROOT, "paddle_ext", "p3d_paddle_ops.cc")).read()
    for op in ("hard_voxelize", "boxes_iou_bev_gpu", "boxes_overlap_bev_gpu", "nms_gpu", "nms_normal_gpu",
               "centerpoint_postprocess", "bev_pool_v2", "bev_pool_v2_bkwd",
               # arithmetic that lives inside PaddlePaddle in the reference: new op names, same registration style
               "p3d_scatter_dense", "p3d_sparse_subm_rulebook", "p3d_sparse_conv_rulebook", "p3d_sparse_gather_gemm"):
        assert "PD_BUILD_OP(%s)" % op in src
