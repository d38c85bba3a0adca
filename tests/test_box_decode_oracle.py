"""CPU: the known-answer NMS inputs of tests/nms_chains.py against the oracle's O(n^2) NMS, and the word-boundary
crossings the GPU tests rely on."""
import numpy as np
import pytest

import nms_chains


def _crossings(lens):
    """Parities of (word boundary - chain start) over every chain that crosses a 64-box word boundary."""
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    return [(b - s) % 2 for s, L in zip(starts, lens) for b in range((s // 64 + 1) * 64, s + L, 64)]


@pytest.mark.parametrize("normal", [False, True])
@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 127, 128, 129, 300])
def test_known_answers_match_oracle_nms(oracle_mod, n, normal):
    cases = [nms_chains.chains(nms_chains.chain_lengths(n, seed, seed % 2)) for seed in range(4)]
    cases += [nms_chains.chains([n]), nms_chains.disjoint(n), nms_chains.identical(n)]
    for boxes, want in cases:
        keep, nk = oracle_mod.nms(boxes, nms_chains.THR, normal)
        assert np.array_equal(keep[:nk], want)


@pytest.mark.parametrize("parity", [0, 1])
def test_chains_cross_word_boundaries(parity):
    """The first crossing has the requested parity at every size from 65 on; the sizes of 4095 and more cross at both
    parities and have chains that end exactly on a boundary."""
    for k in (2, 3, 64, 781):
        for n in (64 * k - 1, 64 * k, 64 * k + 1):
            lens = nms_chains.chain_lengths(n, n, parity)
            assert lens.sum() == n and lens.min() >= 1
            par = _crossings(lens)
            assert par[0] == parity, (n, par)
            if k >= 64:
                ends = np.cumsum(lens)
                assert set(par) == {0, 1} and (ends[:-1] % 64 == 0).any(), n


def test_chain_overlaps(oracle_mod):
    """Neighbours overlap well above the threshold; boxes two apart do not touch; disjoint boxes never overlap."""
    boxes, _ = nms_chains.chains([3])
    iou = oracle_mod.boxes_iou_bev(boxes, boxes)
    assert iou[0, 1] > 2 * nms_chains.THR and iou[1, 2] > 2 * nms_chains.THR and iou[0, 2] == 0
    boxes, _ = nms_chains.disjoint(600)
    iou = oracle_mod.boxes_iou_bev(boxes, boxes)
    assert (iou[~np.eye(600, dtype=bool)] == 0).all()
