"""fp32 restatements and small references for the LiDAR front-end kernels (tests/test_gpu_lidar_front_end.py):

- voxel_mean_f32: the mean of `vox_mean_kernel` / `voxel_mean_kernel` (csrc/voxelize.cu) in the kernels' own order:
  start at +0, add the kept points in slot order in fp32, then one IEEE division by the count.  mean_bound is the a-priori
  distance of that value from the fp64 mean.
- scatter_dense: p3d_scatter_dense's canvas [B, C, D, ny, nx] (csrc/scatter.cu): the row of the highest index among the
  in-range rows of a cell wins, every other element is 0.
- rows_to_pixel_h16: p3d_sparse_rows_to_pixel_h16's pixel image from fp16-pair rows, as uint16 bit patterns.
- nbr_map: the neighbour map [n_out, K] of a sparse conv (tap k = (dz kH + dy) kW + dx, the weight layout
  [kD, kH, kW, Cin, Cout] of oracle.sparse_conv3d) for given input and output sites.
- pfn_bound: the a-priori error of the one-layer pillar encoder (csrc/pillar_encoder.cu) from the fp32 rounding of the
  decoration, the fp32 dot products and the folded BatchNorm.

Everything here is numpy; tests/test_lidar_front_end_oracle.py checks it on the CPU."""
import numpy as np

U32 = 2.0 ** -24  # unit roundoff of fp32


# ------------------------------------------------------------------------------------------------- voxel mean
def voxel_mean_f32(voxels, npv, nv):
    """voxels [V, P, F] zero-padded (hard_voxelize's layout), npv [V]; rows >= nv are 0.  Slot k of voxel v takes part
    iff k < npv[v]; adding the zero padding instead would give the same bits (s + 0 == s for s != -0, and a sum started
    at +0 never becomes -0 in round-to-nearest)."""
    voxels = np.asarray(voxels, np.float32)
    V, P, F = voxels.shape
    npv = np.asarray(npv, np.int64)
    s = np.zeros((V, F), np.float32)
    for k in range(P):
        s = np.where((k < npv)[:, None], (s + voxels[:, k, :]).astype(np.float32), s)
    cnt = np.maximum(npv, 1).astype(np.float32)[:, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = (s / cnt).astype(np.float32)
    mean[nv:] = 0.0
    return mean


def voxel_mean_f64(voxels, npv, nv):
    v = np.asarray(voxels, np.float64)[:nv]
    return v.sum(1) / np.asarray(npv[:nv], np.float64)[:, None]


def mean_bound(voxels, npv, nv, P, got):
    """|fp32 mean - fp64 mean| <= P 2^-24 sum|x| / cnt + 1/2 ulp: the recursive fp32 sum of cnt <= P terms is off by at
    most (cnt - 1) 2^-24 sum|x| (the division by cnt carries that over divided by cnt), the division rounds once."""
    a = np.abs(np.asarray(voxels, np.float64)[:nv]).sum(1)
    cnt = np.asarray(npv[:nv], np.float64)[:, None]
    want = voxel_mean_f64(voxels, npv, nv)
    ulp = np.spacing(np.maximum(np.abs(want), np.abs(np.asarray(got, np.float64)[:nv])).astype(np.float32))
    return P * U32 * a / cnt + 0.5 * ulp.astype(np.float64)


# ------------------------------------------------------------------------------------------------- dense scatter
def scatter_dense(feats, coords, n, batch, D, ny, nx, use_z):
    """feats [cap, C], coords [cap, 4] (b, z, y, x); rows >= n are ignored, rows with any field out of range skipped
    (z is read only with use_z, else 0).  Duplicate cells: the highest row index wins (scatter-overwrite order)."""
    feats = np.asarray(feats, np.float32)
    C = feats.shape[1]
    c = np.asarray(coords, np.int64)[:n]
    z = c[:, 1] if use_z else np.zeros(len(c), np.int64)
    ok = (c[:, 0] >= 0) & (c[:, 0] < batch) & (z >= 0) & (z < D) & (c[:, 2] >= 0) & (c[:, 2] < ny) & (c[:, 3] >= 0) & \
        (c[:, 3] < nx)
    rows = np.nonzero(ok)[0]
    cell = ((c[rows, 0] * D + z[rows]) * ny + c[rows, 2]) * nx + c[rows, 3]
    winner = np.full(batch * D * ny * nx, -1, np.int64)
    np.maximum.at(winner, cell, rows)
    out = np.zeros((batch, D * ny * nx, C), np.float32)
    live = winner >= 0
    out.reshape(-1, C)[live] = feats[winner[live]]
    return np.ascontiguousarray(out.transpose(0, 2, 1)).reshape(batch, C, D, ny, nx)


# ------------------------------------------------------------------------------------------------- rows -> pixel rows
def rows_to_pixel_h16(rows_u16, coords, n, C, batch, D, ny, nx):
    """rows_u16 [cap, 2 C] uint16 (fp16-pair rows: groups of 32 channels, [hi 32 | lo' 32] each); coords [cap, 4]
    (b, z, y, x), unique among the in-range rows < n.  Returns [batch * ny * nx, 2 D C] uint16: row r at pixel (b, y, x),
    channels z C .. z C + C - 1, i.e. halfs 2 z C .. 2 (z + 1) C (C % 32 == 0 keeps the groups aligned); zeros elsewhere."""
    rows_u16 = np.asarray(rows_u16, np.uint16)
    c = np.asarray(coords, np.int64)[:n]
    ok = (c[:, 0] >= 0) & (c[:, 0] < batch) & (c[:, 1] >= 0) & (c[:, 1] < D) & (c[:, 2] >= 0) & (c[:, 2] < ny) & \
        (c[:, 3] >= 0) & (c[:, 3] < nx)
    out = np.zeros((batch * ny * nx, D, 2 * C), np.uint16)
    r = np.nonzero(ok)[0]
    px = (c[r, 0] * ny + c[r, 2]) * nx + c[r, 3]
    assert len(np.unique(px * D + c[r, 1])) == len(r), "rows_to_pixel_h16 has no defined winner for duplicate sites"
    out[px, c[r, 1]] = rows_u16[r]
    return out.reshape(batch * ny * nx, 2 * D * C)


def zc_order(canvas):
    """[B, C, D, H, W] -> [B, D C, H, W]: the (c, z) channel order of to_dense + transpose + reshape permuted to the
    (z, c) order of the pixel rows (dense_head.py, SparseCooTensor.to_pixel_h16)."""
    B, C, D, H, W = canvas.shape
    return np.ascontiguousarray(np.asarray(canvas).transpose(0, 2, 1, 3, 4)).reshape(B, D * C, H, W)


# ------------------------------------------------------------------------------------------------- sparse conv
def _keys(c, spatial):
    D, H, W = spatial
    c = np.asarray(c, np.int64)
    return ((c[:, 0] * (D + 2) + c[:, 1] + 1) * (H + 2) + c[:, 2] + 1) * (W + 2) + c[:, 3] + 1


def nbr_map(in_coords, out_coords, spatial, ksize, stride=(1, 1, 1), padding=(0, 0, 0)):
    """nbr[o][k] = the input row at out_coords[o] * stride - padding + (dz, dy, dx), k = (dz kH + dy) kW + dx, or -1."""
    in_coords = np.asarray(in_coords, np.int64)
    out_coords = np.asarray(out_coords, np.int64)
    kd, kh, kw = ksize
    order = np.argsort(_keys(in_coords, spatial), kind="stable")
    sk = _keys(in_coords, spatial)[order]
    nbr = np.full((len(out_coords), kd * kh * kw), -1, np.int32)
    base = out_coords[:, 1:] * np.asarray(stride) - np.asarray(padding)
    k = 0
    for dz in range(kd):
        for dy in range(kh):
            for dx in range(kw):
                p = base + np.asarray([dz, dy, dx])
                inside = np.all((p >= 0) & (p < np.asarray(spatial)), 1)
                q = np.concatenate([out_coords[:, :1], p], 1)
                key = _keys(np.where(inside[:, None], q, 0), spatial)
                pos = np.clip(np.searchsorted(sk, key), 0, max(len(sk) - 1, 0))
                hit = inside & (len(sk) > 0) & (sk[pos] == key) if len(sk) else np.zeros(len(q), bool)
                nbr[hit, k] = order[pos[hit]]
                k += 1
    return nbr


def gather_conv_f64(feats, nbr, weight):
    """out[o] = sum_k feats[nbr[o][k]] @ W[k] in fp64; weight [K, Cin, Cout] (or Paddle's [kD, kH, kW, Cin, Cout])."""
    f = np.asarray(feats, np.float64)
    w = np.asarray(weight, np.float64)
    w = w.reshape(-1, w.shape[-2], w.shape[-1])
    out = np.zeros((len(nbr), w.shape[-1]))
    for k in range(w.shape[0]):
        src = nbr[:, k]
        hit = src >= 0
        out[hit] += f[src[hit]] @ w[k]
    return out


# ------------------------------------------------------------------------------------------------- pillar encoder
def pfn_bound(voxels, npv, coors, weight, scale, shift, voxel_size, point_cloud_range):
    """Per (pillar, channel) a-priori bound on |kernel - fp64 oracle| for the one-layer PillarFeatureNet with the folded
    (scale, shift) the kernel reads (fp32).  The oracle's fp64 BatchNorm differs from them by at most 2^-24 |scale| and
    2^-24 |shift| (one rounding each).  Per decorated row m and feature d, the kernel's input error delta[m, d] is
      d < F               0 (a copy);
      xyz - mean          |mean error| + 1/2 ulp(value): the fp32 mean of cnt <= M points is off by
                          M 2^-24 sum|x| / cnt + 1/2 ulp(mean);
      xy - centre         centre = c v + off in fp32 (FMA or not: at most two roundings of 1/2 ulp(|c v| + |off|)),
                          then 1/2 ulp(value).
    The fp32 dot product over D = F + 5 terms adds D 2^-24 sum_d |x_d w_d|, the fmaf epilogue 1/2 ulp; ReLU and the max
    over rows are 1-Lipschitz, so the channel's bound is the largest row bound."""
    v = np.asarray(voxels, np.float64)
    n, m, f = v.shape
    cnt = np.asarray(npv, np.float64).reshape(-1, 1)
    live = (np.arange(m)[None, :] < cnt)
    ulp = lambda x: np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)  # noqa: E731
    pmean = v[:, :, :3].sum(1) / cnt
    mean_err = m * U32 * np.abs(v[:, :, :3]).sum(1) / cnt + 0.5 * ulp(np.abs(pmean) * (1 + m * U32))
    clus = v[:, :, :3] - pmean[:, None, :]
    d_clus = mean_err[:, None, :] + 0.5 * ulp(np.abs(clus) + mean_err[:, None, :])
    vx, vy = float(voxel_size[0]), float(voxel_size[1])
    xo = np.float32(np.float32(vx) / 2 + np.float32(point_cloud_range[0]))
    yo = np.float32(np.float32(vy) / 2 + np.float32(point_cloud_range[1]))
    c = np.asarray(coors, np.float64)
    cv = np.stack([c[:, 3] * np.float32(vx), c[:, 2] * np.float32(vy)], 1)
    cen = cv + np.asarray([xo, yo], np.float64)
    cen_err = ulp(np.abs(cv) + np.abs(cen))
    cent = v[:, :, :2] - cen[:, None, :]
    d_cent = cen_err[:, None, :] + 0.5 * ulp(np.abs(cent) + cen_err[:, None, :])
    delta = np.concatenate([np.zeros((n, m, f)), d_clus, d_cent], -1) * live[:, :, None]
    feats = np.concatenate([v, clus, cent], -1) * live[:, :, None]
    w = np.abs(np.asarray(weight, np.float64))
    sc = np.abs(np.asarray(scale, np.float64))
    sh = np.abs(np.asarray(shift, np.float64))
    acc = np.abs(feats) @ w                               # sum_d |x_d w_d| per row and channel
    row = sc * (delta @ w + (f + 5 + 2) * U32 * acc) + U32 * (sc * acc + sh)
    row = row + 0.5 * ulp(sc * acc + sh)
    return row.max(1) + U32 * sh  # padding rows: ReLU(shift) in fp32 against the oracle's fp64 shift
