"""CPU: the streaming multi-sweep input (paddle3d_b200/sweep_ring.py) - the ring's slot / frame schedule, the pose ->
ref_from_curr / time-lag arithmetic - and the array-level host merge io.merge_sweeps against the reference golden."""
import numpy as np
import pytest

from conftest import golden
from paddle3d_b200 import io as p3d_io
from paddle3d_b200 import sweep_ring, synth


@pytest.mark.parametrize("K,slots", [(1, 1), (3, 3), (3, 4), (10, 11), (10, 14)])
@pytest.mark.parametrize("n", [0, 1, 5, 37])
def test_ring_schedule_invariants(n, K, slots):
    ops = list(sweep_ring.schedule(n, K, slots))
    content = {}       # slot -> sweep held
    readers = {}       # sweep -> frames that read it
    frames = []
    for op in ops:
        if op[0] == "push":
            _, j, slot, wait = op
            assert slot == j % slots
            old = content.get(slot)
            # the push waits for exactly the last frame that read the sweep it overwrites
            assert wait == (max(readers[old]) if old is not None and readers.get(old) else None)
            if wait is not None:
                assert wait < j and wait in frames  # an event that has been recorded already
                # with slots = K + lanes, that frame is at least `lanes` frames old: its result was read back already
                assert wait <= j - (slots - K) - 1
            content[slot] = j
        else:
            _, j, reads = op
            assert [s for s, _ in reads] == list(range(j, max(0, j - K + 1) - 1, -1))  # key first, then newest first
            for s, sl in reads:
                assert content[sl] == s, "frame %d reads slot %d, which holds sweep %s" % (j, sl, content.get(sl))
                readers.setdefault(s, []).append(j)
            frames.append(j)
    assert frames == list(range(n))
    with pytest.raises(ValueError):
        list(sweep_ring.schedule(3, K + 1, K))


def test_frame_sweeps_at_stream_start():
    assert sweep_ring.frame_sweeps(0, 10) == [0]
    assert sweep_ring.frame_sweeps(3, 10) == [3, 2, 1, 0]
    assert sweep_ring.frame_sweeps(12, 10) == list(range(12, 2, -1))
    assert sweep_ring.frame_sweeps(12, 10, first=7) == [12, 11, 10, 9, 8, 7]


def test_pose_arithmetic():
    """ref_from_curr = inv(global_from_key) @ global_from_sweep: a sweep point moved by it lands where the same world
    point is seen from the key pose; lag = t_key - t_sweep."""
    seq = synth.sweep_sequence(4, 0, points_per_sweep=2000)
    (ck, pk, tk), (cs, ps, ts) = seq[3], seq[0]
    m = sweep_ring.ref_from_curr(pk, ps)
    assert m.dtype == np.float64 and np.allclose(m[3], [0, 0, 0, 1])
    xyz1 = np.hstack([cs[:, :3].astype(np.float64), np.ones((len(cs), 1))])
    world = xyz1 @ ps.T
    assert np.allclose(xyz1 @ m.T, world @ np.linalg.inv(pk).T, atol=1e-9)
    assert np.allclose(sweep_ring.ref_from_curr(pk, pk), np.eye(4), atol=1e-12)
    assert np.isclose(tk - ts, 0.15)
    # the ego moves and turns between sweeps: the transform is neither the identity nor a pure translation
    assert abs(m[0, 1]) > 1e-3 and np.linalg.norm(m[:3, 3]) > 1.0
    assert all(c.shape[1] == 5 and c.dtype == np.float32 for c, _, _ in seq)


def test_merge_sweeps_arrays_match_reference_golden():
    """io.merge_sweeps (the host oracle of ops.sweep_merge) on the golden's raw arrays, in the golden's order."""
    g = golden("sweeps.npz")
    sweeps = [(g["cloud1"], g["mat0"], float(g["lags"][0])), (g["cloud2"], None, float(g["lags"][1])),
              (g["cloud3"], g["mat2"], float(g["lags"][2]))]
    out = p3d_io.merge_sweeps(g["cloud0"], sweeps, use_dim=[0, 1, 2, 4], use_time_lag=True, sweep_remove_radius=1,
                              order=g["order"])
    assert out.dtype == np.float32 and np.array_equal(out, g["merged"])
    # the inputs are not modified
    assert np.array_equal(sweeps[0][0], g["cloud1"]) and np.array_equal(sweeps[2][0], g["cloud3"])
    assert np.array_equal(p3d_io.merge_sweeps(g["cloud0"]), g["cloud0"])
