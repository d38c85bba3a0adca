"""CPU: the frames-in-flight schedule (frame.in_flight) as CenterPointSweep.infer_many / infer_stream and a single
frame's infer_many / infer_stream run it, on stub lanes that record what they are asked to do instead of running a
frame: the recorded order is CenterPointSweep.plan's, and a (lane, slot) skips the wait for its staging buffer exactly on
its first use."""
import pytest

from paddle3d_b200.frame import CapturedFrame
from paddle3d_b200.pipeline import CenterPointSweep


class _Ring:
    def __init__(self):
        self.pushed = 0

    def reset(self):
        self.pushed = 0

    def push(self, cloud, pose, t):
        self.pushed += 1
        return self.pushed - 1


class _Lane(CapturedFrame):
    def __init__(self, idx, log, ring):
        self.idx, self.log, self.ring, self.graph = idx, log, ring, object()
        self.frame_of, self.used = {}, set()

    def prepare_sweep(self):
        return self

    def _submit(self, pts, k, first_use):
        assert first_use == ((self.idx, k) not in self.used)
        self.used.add((self.idx, k))
        self._submit_sweep(pts, k)

    def _submit_sweep(self, j, k):
        assert k not in self.frame_of, "slot resubmitted before its result was read"
        self.frame_of[k] = j
        self.log.append(("submit", j, self.idx, k))

    def _result(self, k):
        self.log.append(("result", self.frame_of.pop(k), self.idx, k))
        return k


def _sweep(lanes, log, ring):
    sweep = CenterPointSweep.__new__(CenterPointSweep)
    sweep.lanes = [_Lane(i, log, ring) for i in range(lanes)]
    return sweep


@pytest.mark.parametrize("lanes", [1, 2, 3, 4])
def test_infer_many_and_stream_follow_plan(lanes):
    for n in range(17):
        want = list(CenterPointSweep.plan(n, lanes))
        runs = {"CenterPointSweep.infer_many": lambda s, ring: s.infer_many(range(n)),
                "CenterPointSweep.infer_stream": lambda s, ring: s.infer_stream((j, None, 0.0) for j in range(n))}
        if lanes == 1:
            runs["CapturedFrame.infer_many"] = lambda s, ring: s.lanes[0].infer_many(range(n))
            runs["CapturedFrame.infer_stream"] = lambda s, ring: s.lanes[0].infer_stream((j, None, 0.0) for j in range(n))
        for name, run in runs.items():
            log, ring = [], _Ring()
            results = list(run(_sweep(lanes, log, ring), ring))
            assert log == want, (name, n)
            assert results == [o[3] for o in want if o[0] == "result"], (name, n)
