"""CPU suite: the row order of a strided sparse conv's output, restated in numpy.

A strided level's rows are its output sites in first-appearance order: walk the input rows in row order and, within a
row, the taps in tap order (k = (kz kH + ky) kW + kx), and append each site the first time it is generated.  A row
whose coordinate a later row repeats generates no sites (the later row stands for the coordinate), and neither does a
row outside the input grid.  first_appearance_sites restates that order and the strided neighbour map in that order;
the tests below pin it on hand-built cases, and against the order-free references (test_gpu_centerpoint_full_size's
strided_sites for the set, lidar_front_end_oracle.nbr_map for the taps) on a random one.  The GPU tests
(test_gpu_reproducible_frames) hold the rulebook kernels to it."""
import numpy as np

import lidar_front_end_oracle as lfo
from test_gpu_centerpoint_full_size import strided_sites


def _lin(c, dims):
    """Linear key of [n, 4] (b, z, y, x) over (D, H, W)."""
    return ((c[:, 0] * dims[0] + c[:, 1]) * dims[1] + c[:, 2]) * dims[2] + c[:, 3]


def first_appearance_sites(coords, batch, spatial, ksize, stride, padding):
    """(out_coords [m, 4] int32 in first-appearance order, nbr [m, K] int32, output spatial shape) of a strided conv
    over the input rows coords [n, 4]: nbr[o][k] = the row standing for the input cell o * stride - padding + k, or -1."""
    c = np.asarray(coords, np.int64).reshape(-1, 4)
    sp, k, s, p = (np.asarray(v, np.int64) for v in (spatial, ksize, stride, padding))
    osp = (sp + 2 * p - k) // s + 1
    K = int(np.prod(k))
    inside = (c[:, 0] >= 0) & (c[:, 0] < batch) & (c[:, 1:] >= 0).all(1) & (c[:, 1:] < sp).all(1)
    # the row standing for each coordinate: the last of its rows
    rows = np.nonzero(inside)[0]
    keys = _lin(c[rows], sp)
    last = len(keys) - 1 - np.unique(keys[::-1], return_index=True)[1]
    canon_rows, canon_keys = rows[last], keys[last]  # sorted by key
    canon = np.zeros(len(c), bool)
    canon[canon_rows] = True
    taps = [(dz, dy, dx) for dz in range(k[0]) for dy in range(k[1]) for dx in range(k[2])]
    # cand[i, k]: the linear output key of row i under tap k, or -1; read row-major, that is (i, k) order
    cand = np.full((len(c), K), -1, np.int64)
    for t, d in enumerate(taps):
        o = c[:, 1:] + p - np.asarray(d)
        ok = canon & (o >= 0).all(1) & (o % s == 0).all(1)
        o = o // s
        ok &= (o < osp).all(1)
        cand[ok, t] = _lin(np.concatenate([c[ok, :1], o[ok]], 1), osp)
    flat = cand.ravel()
    flat = flat[flat >= 0]
    u, first = np.unique(flat, return_index=True)
    u = u[np.argsort(first)]
    vol = int(np.prod(osp))
    out = np.stack([u // vol, u // (osp[1] * osp[2]) % osp[0], u // osp[2] % osp[1], u % osp[2]], 1)
    nbr = np.full((len(out), K), -1, np.int32)
    for t, d in enumerate(taps):
        q = out[:, 1:] * s - p + np.asarray(d)
        ok = (q >= 0).all(1) & (q < sp).all(1)
        key = _lin(np.concatenate([out[:, :1], np.where(ok[:, None], q, 0)], 1), sp)
        pos = np.clip(np.searchsorted(canon_keys, key), 0, max(len(canon_keys) - 1, 0))
        hit = ok & (canon_keys[pos] == key) if len(canon_keys) else np.zeros(len(out), bool)
        nbr[hit, t] = canon_rows[pos[hit]]
    return out.astype(np.int32), nbr, osp


def _rows(*xs):
    return np.asarray(xs, np.int32).reshape(-1, 4)


def test_batch_two_stride_two():
    """Batch 2, a 1 x 3 window of stride 2 and padding 1 along x: the sites come in row order, within a row in tap
    order (x = 5 makes site 3 under tap 0 before site 2 under tap 2), not sorted."""
    coords = _rows((1, 0, 0, 5), (0, 0, 0, 5), (1, 0, 0, 0), (1, 0, 0, 3))
    out, nbr, osp = first_appearance_sites(coords, 2, (1, 1, 8), (1, 1, 3), (1, 1, 2), (0, 0, 1))
    assert list(osp) == [1, 1, 4]
    assert out.tolist() == [[1, 0, 0, 3], [1, 0, 0, 2], [0, 0, 0, 3], [0, 0, 0, 2], [1, 0, 0, 0], [1, 0, 0, 1]]
    assert nbr.tolist() == [[0, -1, -1], [3, -1, 0], [1, -1, -1], [-1, -1, 1], [-1, 2, -1], [-1, -1, 3]]


def test_extra_conv_geometry():
    """SparseResNet3D's extra conv: kernel (3, 1, 1), stride (2, 1, 1), no padding."""
    coords = _rows((0, 4, 0, 0), (0, 1, 0, 0), (0, 2, 0, 0))
    out, nbr, osp = first_appearance_sites(coords, 1, (5, 1, 1), (3, 1, 1), (2, 1, 1), (0, 0, 0))
    assert list(osp) == [2, 1, 1]
    assert out.tolist() == [[0, 1, 0, 0], [0, 0, 0, 0]]
    assert nbr.tolist() == [[2, -1, 0], [-1, 1, 2]]


def test_padding_zero_one_one():
    """The last stage's geometry, kernel 3, stride 2, padding (0, 1, 1): the row (2, 1, 1) makes four sites under taps
    18, 20, 24, 26; two of them are new."""
    coords = _rows((0, 1, 2, 0), (0, 0, 0, 0), (0, 2, 1, 1))
    out, nbr, osp = first_appearance_sites(coords, 1, (3, 3, 3), (3, 3, 3), (2, 2, 2), (0, 1, 1))
    assert list(osp) == [1, 2, 2]
    assert out.tolist() == [[0, 0, 1, 0], [0, 0, 0, 0], [0, 0, 1, 1], [0, 0, 0, 1]]
    assert nbr[0, 13] == 0 and nbr[0, 20] == 2 and (nbr[0] >= 0).sum() == 2
    assert nbr[1, 4] == 1 and nbr[1, 26] == 2 and (nbr[1] >= 0).sum() == 2
    assert nbr[2, 18] == 2 and (nbr[2] >= 0).sum() == 1
    assert nbr[3, 24] == 2 and (nbr[3] >= 0).sum() == 1


def test_duplicate_coordinates():
    """Row 2 repeats row 0's coordinate: row 0 generates no site, row 2 stands for the coordinate in the map."""
    coords = _rows((0, 0, 0, 5), (0, 0, 0, 0), (0, 0, 0, 5), (0, 0, 0, 3))
    out, nbr, _ = first_appearance_sites(coords, 1, (1, 1, 8), (1, 1, 3), (1, 1, 2), (0, 0, 1))
    assert out[:, 3].tolist() == [0, 3, 2, 1]
    assert nbr.tolist() == [[-1, 1, -1], [2, -1, -1], [3, -1, 2], [-1, -1, 3]]


def test_rows_outside_the_grid():
    """Rows outside the input grid (x = 9 and x = -1 of 8, batch 1 of 1) generate no sites and are in no map."""
    coords = _rows((0, 0, 0, 9), (0, 0, 0, 5), (0, 0, 0, -1), (1, 0, 0, 3), (0, 0, 0, 3))
    out, nbr, _ = first_appearance_sites(coords, 1, (1, 1, 8), (1, 1, 3), (1, 1, 2), (0, 0, 1))
    assert out.tolist() == [[0, 0, 0, 3], [0, 0, 0, 2], [0, 0, 0, 1]]
    assert nbr.tolist() == [[1, -1, -1], [4, -1, 1], [-1, -1, 4]]


def test_empty_input():
    out, nbr, _ = first_appearance_sites(np.zeros((0, 4), np.int32), 1, (9, 9, 9), (3, 3, 3), (2, 2, 2), (1, 1, 1))
    assert out.shape == (0, 4) and nbr.shape == (0, 27)


def test_random_sites_match_the_order_free_references():
    """Two batches of random sites: the same set as strided_sites, the same taps as lfo.nbr_map, and every site's first
    generating (row, tap) pair comes after the previous site's."""
    rng = np.random.default_rng(5)
    spatial = (7, 12, 11)
    occ = rng.random((2,) + spatial) < 0.2
    coords = np.argwhere(occ).astype(np.int32)
    coords = coords[rng.permutation(len(coords))]
    for k, s, p in (((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (0, 1, 1)), ((3, 1, 1), (2, 1, 1), (0, 0, 0))):
        out, nbr, osp = first_appearance_sites(coords, 2, spatial, k, s, p)
        want, wosp = strided_sites(coords, spatial, k, s, p)
        assert list(osp) == list(wosp) and len(out) == len(want)
        assert np.array_equal(np.sort(_lin(out, osp)), _lin(want, osp))
        assert np.array_equal(nbr, lfo.nbr_map(coords, out, spatial, k, s, p))
        # a site's first generating (row, tap) pair is its smallest (nbr[o][t], t): under tap t, row nbr[o][t] sees o
        K = int(np.prod(k))
        gen = np.where(nbr >= 0, nbr.astype(np.int64) * K + np.arange(K)[None, :], 1 << 62).min(1)
        assert (np.diff(gen) > 0).all()
