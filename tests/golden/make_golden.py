"""Generate the committed golden fixtures from the REFERENCE ITSELF (needs a Paddle3D source checkout named by
$P3D_REFERENCE and oracle/_ref built from it; the tests only read the committed .npz files).

  voxelize_*.npz   outputs of the reference's own hard_voxelize_cpu (voxelize_op.cc:84-146, compiled
                   unmodified into oracle/_ref/libp3d_ref_cpu.so) AND of the reference's numba
                   points_to_voxel (paddle3d/transforms/functional.py:118-150, AST-extracted and exec'd —
                   importing the package would import paddle) on seeded inputs; the two must agree.
  iou_bev.npz      boxes_iou_bev_cpu (iou3d_cpu.cpp:241-264, compiled unmodified).
  sweeps.npz       LoadPointCloud.__call__ (paddle3d/transforms/reader.py:116-167, AST-extracted: importing the module
                   would import paddle) on three seeded .bin files; stores the files' contents, the transforms, the
                   sweep order the reference's np.random.choice drew and the merged cloud.

Usage: python tests/golden/make_golden.py
"""
import ast
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from paddle3d_b200 import synth  # noqa: E402

REF = os.environ.get("P3D_REFERENCE", "")  # a Paddle3D source checkout
HERE = os.path.dirname(os.path.abspath(__file__))


def numba_points_to_voxel():
    import numba  # noqa: F401
    src = open(os.path.join(REF, "paddle3d/transforms/functional.py")).read()
    tree = ast.parse(src)
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "points_to_voxel"][0]
    code = ast.get_source_segment(src, fn)
    ns = {"numba": __import__("numba"), "np": np}
    exec(code, ns)
    return ns["points_to_voxel"]


def run_numba(fn, pts, cfg, P, V):
    vs = np.asarray(cfg["voxel_size"], np.float32)
    pcr = np.asarray(cfg["point_cloud_range"], np.float32)
    grid = np.round((pcr[3:] - pcr[:3]) / vs).astype(np.int32)
    voxels = np.zeros((V, P, pts.shape[1]), np.float32)
    coords = np.zeros((V, 3), np.int32)
    npv = np.zeros((V,), np.int32)
    g2v = np.full(tuple(grid[::-1]), -1, np.int32)
    nv = fn(pts, vs, pcr, grid, voxels, coords, npv, g2v, P, V)
    return voxels, coords, npv, np.array([nv], np.int32)


def reference_load_point_cloud():
    """The reference's LoadPointCloud class body (methods only), exec'd without its paddle-importing module."""
    src = open(os.path.join(REF, "paddle3d/transforms/reader.py")).read()
    tree = ast.parse(src)
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "LoadPointCloud"][0]
    code = "class LoadPointCloud:\n" + "\n".join(
        "    " + line for fn in cls.body if isinstance(fn, ast.FunctionDef)
        for line in ast.get_source_segment(src, fn).splitlines())
    import typing
    ns = {"np": np, "Union": typing.Union, "List": typing.List, "Sample": object, "PointCloud": lambda x: x}
    exec(code, ns)
    return ns["LoadPointCloud"]


def make_sweeps_golden():
    import tempfile
    from types import SimpleNamespace as NS
    rng = np.random.default_rng(21)
    clouds = [np.concatenate([rng.uniform(-3, 3, size=(n, 3)), rng.uniform(0, 255, size=(n, 1)),
                              rng.integers(0, 32, size=(n, 1))], 1).astype(np.float32) for n in (500, 400, 300, 350)]
    mats, lags = [], [0.05, 0.1, 0.15]
    for k in range(3):
        a = 0.01 * (k + 1)
        m = np.eye(4)
        m[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
        m[:3, 3] = [0.3 * (k + 1), -0.1 * k, 0.02]
        mats.append(m)
    mats[1] = None  # a sweep without transform
    with tempfile.TemporaryDirectory() as d:
        paths = []
        for i, c in enumerate(clouds):
            paths.append(os.path.join(d, "c%d.bin" % i))
            c.tofile(paths[-1])
        sweeps = [NS(path=paths[i + 1], meta=NS(ref_from_curr=mats[i], time_lag=lags[i])) for i in range(3)]
        sample = NS(modality="lidar", data=None, path=paths[0], sweeps=sweeps)
        cls = reference_load_point_cloud()
        np.random.seed(1)
        order = np.random.choice(3, 3, replace=False)  # what the call below will draw
        np.random.seed(1)
        out = cls(dim=5, use_dim=[0, 1, 2, 4], use_time_lag=True, sweep_remove_radius=1)(sample).data
    np.savez_compressed(os.path.join(HERE, "sweeps.npz"), cloud0=clouds[0], cloud1=clouds[1], cloud2=clouds[2],
                        cloud3=clouds[3], mat0=mats[0], mat2=mats[2], lags=np.asarray(lags), order=order, merged=out)
    print("sweeps", out.shape, out.dtype, "order", order)


def main():
    oracle.build(ref=True)
    make_sweeps_golden()
    p2v = numba_points_to_voxel()
    cases = {
        # name: (cfg, generator, seed, num_points, max_points, max_voxels)
        "c1_uniform": (synth.C1, synth.uniform_cloud, 0, 1000, 32, 40000),
        "c1_dense": (synth.C1, "dense", 5, 1000, 5, 120),                      # many points per cell, cap, P overflow
        "c1_cap": (synth.C1, synth.uniform_cloud, 1, 1000, 2, 300),            # hits the max_voxels cap
        "c2_lidar_small": (synth.C2, synth.lidar_cloud, 2, 4000, 4, 1500),     # over-full cells + cap
        "c3_lidar_small": (synth.C3, synth.lidar_cloud, 3, 6000, 3, 5000),
    }
    for name, (cfg, gen, seed, n, P, V) in cases.items():
        if gen == "dense":
            rng = np.random.default_rng(seed)
            pts = np.concatenate([rng.normal([30, 0, -1], [1.0, 1.0, 0.5], size=(n, 3)), rng.uniform(0, 1, (n, 1))], 1).astype(np.float32)
        else:
            pts = gen(cfg, seed, num_points=n)
        if name == "c2_lidar_small":
            pts = pts[(pts[:, 0] > 0)][:n]
        ref = oracle.ref_hard_voxelize_cpu(pts, cfg["voxel_size"], cfg["point_cloud_range"], P, V)
        nb = run_numba(p2v, pts, cfg, P, V)
        for a, b in zip(ref, nb):
            assert np.array_equal(a, b), "reference C++ and numba voxelizers disagree on %s" % name
        np.savez_compressed(os.path.join(HERE, "voxelize_%s.npz" % name), points=pts,
                            voxel_size=np.asarray(cfg["voxel_size"], np.float32),
                            point_cloud_range=np.asarray(cfg["point_cloud_range"], np.float32),
                            max_points=P, max_voxels=V, voxels=ref[0], coords=ref[1], num_points_per_voxel=ref[2],
                            num_voxels=ref[3])
        print(name, "num_voxels", int(ref[3][0]), "max npv", int(ref[2].max()))
    a = synth.random_boxes(96, 11)
    rng = np.random.default_rng(12)
    b = a[rng.permutation(96)[:80]].copy()
    b[:, :2] += rng.normal(0, 0.8, size=(80, 2)).astype(np.float32)
    b[:, 6] += rng.normal(0, 0.4, size=80).astype(np.float32)
    b[:8] = a[:8]  # identical boxes
    b[8:16] = a[8:16]
    b[8:16, 6] += 1e-3  # nearly identical
    iou = oracle.ref_boxes_iou_bev_cpu(a, b)
    np.savez_compressed(os.path.join(HERE, "iou_bev.npz"), boxes_a=a, boxes_b=b, iou=iou)
    print("iou_bev", iou.shape, "nonzero", float((iou > 0).mean()))


if __name__ == "__main__":
    main()
