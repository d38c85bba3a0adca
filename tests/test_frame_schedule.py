"""CPU: the frames-in-flight schedule (frame.in_flight) as CenterPointSweep.infer_many / infer_stream, a single
frame's infer_many / infer_stream and the BEVDet4D drives' infer_stream run it, on stub lanes that record what they are
asked to do instead of running a frame: the recorded order is CenterPointSweep.plan's (for the drives: item j + 1 staged
before frame j's result is read), and a (lane, staging set) skips the wait for its staging buffers exactly on its first
use (_Upload, standing in for frame.StagedUpload)."""
import numpy as np
import pytest

from paddle3d_b200.bevdet import BEVDet4DFrameHotPath, BEVDet4DJpegHotPath
from paddle3d_b200.frame import CapturedFrame
from paddle3d_b200.pipeline import CenterPointSweep


class _Upload:
    """StagedUpload's bookkeeping without a device: stage() calls fill(k, None) and holds its payload in set k until
    unstage(k) returns it."""

    def __init__(self):
        self.held, self.used = {}, set()

    def stage(self, k, fill, first_use):
        assert first_use == (k not in self.used), "set %d: first_use=%s" % (k, first_use)
        assert k not in self.held, "staging set %d refilled before it was consumed" % k
        self.used.add(k)
        self.held[k] = fill(k, None)

    def unstage(self, k, stream):
        return self.held.pop(k)


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
        self.idx, self.log, self.ring, self.graph, self.stream = idx, log, ring, object(), None
        self.frame_of, self._upload = {}, _Upload()

    def prepare_sweep(self):
        return self

    def _submit(self, pts, k, first_use):
        self._upload.stage(k, lambda dev, host: pts, first_use)
        self._submit_sweep(self._upload.unstage(k, self.stream), k)

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


class _Drive:
    """A BEVDet4D lane's infer_stream on stubs: item j = (j, identity poses, cam2imgs j); test_mats returns cam2imgs, so
    a launched step names its item."""

    def __init__(self, log):
        self.log, self.graphs, self._upload, self.running = log, {"start": None}, _Upload(), []
        self.model, self.slot, self.done, self.stream = self, self, None, None

    @staticmethod
    def test_mats(sensor2keyego, cam2imgs, bda):
        return cam2imgs

    def _fill(self, payload, dev, host):
        self.log.append(("stage", payload, dev))
        return payload

    def _launch_step(self, step, k):
        j = int(step[0][0])
        assert self._upload.unstage(k, self.stream) == j and step[2] == (j == 0)
        self.running.append(j)
        self.log.append(("launch", j, k))

    def read(self, check_status, copied, clone=False):
        assert clone and len(self.running) == 1
        self.log.append(("result", self.running.pop()))
        return self.log[-1][1]


@pytest.mark.parametrize("cls", [BEVDet4DFrameHotPath, BEVDet4DJpegHotPath])
def test_drive_stages_next_item_during_frame(cls):
    stub = type("_Stub", (_Drive, cls), {})
    eye = np.eye(4)[None]
    for n in range(7):
        want = []
        for j in range(n):
            want += [("stage", 0, 0), ("launch", 0, 0)] if j == 0 else []
            want += [("stage", j + 1, (j + 1) & 1)] if j + 1 < n else []
            want += [("result", j)]
            want += [("launch", j + 1, (j + 1) & 1)] if j + 1 < n else []
        log = []
        lane = stub(log)
        assert list(lane.infer_stream((j, eye, eye, j) for j in range(n))) == list(range(n)), n
        assert log == want, n
