"""Input-side data format of the hot path (SURVEY.md §8f-4): nuScenes/KITTI `.bin` point files and the multi-sweep
merge that produces the [N, F] fp32 cloud `hard_voxelize` consumes.

Host code (numpy), a restatement of `paddle3d/transforms/reader.py:91-167` (`LoadPointCloud`): same column selection,
same close-point removal per sweep, same homogeneous transform into the reference frame, same time-lag column. The one
deliberate difference: the reference visits the sweeps in a random permutation (`np.random.choice`, reader.py:133-134);
here the order is an explicit argument (default: as given), so that a frame is reproducible.
"""
import numpy as np


def read_bin(path, dim, use_dim=None):
    """[N, dim] fp32 points of a `.bin` file (reader.py:123-126); `use_dim` = int (first k columns) or a list."""
    return select_columns(np.fromfile(path, np.float32).reshape(-1, int(dim)), use_dim)


class Sweep:
    """One earlier sweep: file path, 4x4 (or 3x4) transform into the key frame's coordinates or None, time lag [s]."""

    def __init__(self, path, ref_from_curr=None, time_lag=0.0):
        self.path, self.ref_from_curr, self.time_lag = path, ref_from_curr, time_lag


def select_columns(data, use_dim):
    """Columns of [N, dim] rows as read_bin selects them: `use_dim` = None (all), int (first k columns) or a list."""
    if use_dim is None:
        return data
    cols = list(range(use_dim)) if isinstance(use_dim, (int, np.integer)) else list(use_dim)
    return data[:, cols]


def load_point_cloud(path, dim, use_dim=None, use_time_lag=False, sweeps=(), sweep_remove_radius=1.0, order=None):
    """Key-frame cloud + sweeps -> [N, F] fp32 (F = len(use_dim) + use_time_lag).

    sweeps: sequence of `Sweep`; order: permutation of range(len(sweeps)) (None = as given)."""
    clouds = [(read_bin(sw.path, dim), sw.ref_from_curr, sw.time_lag) for sw in sweeps]
    return merge_sweeps(read_bin(path, dim), clouds, use_dim, use_time_lag, sweep_remove_radius, order)


def merge_sweeps(key, sweeps=(), use_dim=None, use_time_lag=False, sweep_remove_radius=1.0, order=None):
    """The array half of load_point_cloud: raw [n, dim] fp32 rows of the key sweep and of each earlier sweep -> [N, F].

    sweeps: sequence of (cloud [n_i, dim] fp32, ref_from_curr (4x4 / 3x4) or None, time_lag) tuples;
    order: permutation of range(len(sweeps)) (None = as given).  The host oracle of ops.sweep_merge."""
    data = select_columns(np.asarray(key, np.float32), use_dim)
    if use_time_lag:  # the key frame's own points carry lag 0 (reader.py:128-130)
        data = np.hstack([data, np.zeros((data.shape[0], 1), dtype=data.dtype)])
    if len(sweeps) == 0:
        return data
    idx = range(len(sweeps)) if order is None else [int(i) for i in order]
    if sorted(idx) != list(range(len(sweeps))):
        raise ValueError("order must be a permutation of the sweep indices")
    parts = [data]
    for i in idx:
        cloud, ref_from_curr, time_lag = sweeps[i]
        # `use_dim` falsy (None, 0, []) keeps all columns in the sweep branch of the reference (reader.py:139-140)
        pts = select_columns(np.asarray(cloud, np.float32), use_dim if use_dim else None).T
        # drop the points inside the |x| < r and |y| < r square around the sensor (reader.py:143-150)
        close = np.logical_and(np.abs(pts[0, :]) < sweep_remove_radius, np.abs(pts[1, :]) < sweep_remove_radius)
        pts = pts[:, np.logical_not(close)]
        if ref_from_curr is not None:  # homogeneous transform, computed in float64 (reader.py:153-157)
            m = np.asarray(ref_from_curr)
            pts[:3, :] = m.dot(np.vstack((pts[:3, :], np.ones(pts.shape[1]))))[:3, :]
        pts = pts.T
        if use_time_lag:
            lag = time_lag * np.ones((pts.shape[0], 1)).astype(pts.dtype)
            pts = np.hstack([pts, lag])
        parts.append(pts)
    return np.concatenate(parts, axis=0)
