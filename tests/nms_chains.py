"""Known-answer inputs for the greedy NMS (p3d_nms / nms_greedy_cta) at sizes the O(n^2) oracle cannot afford.

Boxes are unit squares at heading 0, given in score order (index 0 first).  In a chain, consecutive boxes sit 0.625 apart
along x, so neighbours overlap by 0.375 (IoU 0.375 / 1.625 = 0.23, axis-aligned or rotated alike) and boxes two apart
are 0.25 apart and never touch.  Chains sit 4 apart in y.  With an IoU threshold of 0.1 the greedy pass keeps the first
box of a chain, which suppresses the second, keeps the third, and so on: the kept boxes are the even positions of every
chain, found in O(n).  Every coordinate is a binary fraction, so both sides compute the same IoUs."""
import numpy as np

THR = 0.1
STEP = 0.625


def _boxes(xy):
    b = np.zeros((len(xy), 7), np.float32)
    b[:, :2] = xy
    b[:, 2] = -1.0
    b[:, 3:6] = (1.0, 1.0, 1.5)
    return b


def chain_lengths(n, seed, parity=0):
    """Chain lengths summing to n.  The second chain crosses the first word boundary (box 64) at an offset of parity
    `parity` from its start (even: box 64 is kept; odd: box 63 suppresses it); after it come random lengths (1 .. 150),
    chains that end exactly on a boundary and chains that cross one."""
    rng = np.random.default_rng(seed)
    lens, pos = [], 0
    for L in (60 - parity, 10):
        if pos < n:
            lens.append(min(L, n - pos))
            pos += lens[-1]
    while pos < n:
        nxt = (pos // 64 + 1) * 64
        r = rng.integers(0, 4)
        if r == 0 and nxt - pos > 1:
            L = nxt - pos                              # ends on the word boundary
        elif r == 1 and nxt - pos > 2:
            L = nxt - pos + int(rng.integers(1, 9))    # crosses it
        else:
            L = int(rng.integers(1, 151))
        L = min(L, n - pos)
        lens.append(L)
        pos += L
    return np.asarray(lens, np.int64)


def chains(lengths):
    """(boxes [n, 7] fp32, expected keep list int32) for chains of the given lengths, laid out in index order."""
    lengths = np.asarray(lengths, np.int64)
    n = int(lengths.sum())
    starts = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    chain = np.repeat(np.arange(len(lengths)), lengths)
    pos = np.arange(n) - starts[chain]
    xy = np.stack([pos * STEP, chain * 4.0], 1)
    return _boxes(xy), np.nonzero(pos % 2 == 0)[0].astype(np.int32)


def disjoint(n):
    """n boxes 2 apart on a 256-wide raster: all kept."""
    i = np.arange(n)
    return _boxes(np.stack([(i % 256) * 2.0, (i // 256) * 2.0], 1)), i.astype(np.int32)


def identical(n):
    """n copies of one box: only index 0 is kept."""
    return _boxes(np.zeros((n, 2))), np.zeros(min(n, 1), np.int32)
