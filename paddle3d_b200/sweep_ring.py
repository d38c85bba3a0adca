"""Streaming multi-sweep input: a device ring of raw LiDAR sweeps and the per-frame descriptor the merge kernel reads.

A sensor delivers one sweep every ~50 ms; a frame of the nuScenes 10-sweep model uses the newest sweep as its key and
the K - 1 previous ones, each moved into the key frame (ref_from_curr = inv(global_from_key) @ global_from_sweep) with a
time-lag column (t_key - t_sweep).  Each pushed sweep is copied once into a slot of the ring; every frame only uploads
its ~1 KB descriptor, and ops.sweep_merge builds the merged cloud on the device.

A slot is reused only after the last frame that reads it has finished: schedule() is the slot / frame order as a pure
function (tests/test_sweep_ring.py checks its invariants without a GPU) and SweepRing.push waits on the event of that
frame on the copy stream.  With slots = K + lanes, that frame's result has already been read back by the time the slot
is reused, so the wait never stalls the copy stream.
"""
import numpy as np

from .ops import sweep_merge as sm


def ref_from_curr(global_from_key, global_from_curr):
    """4x4 float64 transform from a sweep's sensor frame into the key sweep's sensor frame."""
    return np.linalg.inv(np.asarray(global_from_key, np.float64)) @ np.asarray(global_from_curr, np.float64)


def frame_sweeps(j, max_sweeps, first=0):
    """Sweeps of the frame keyed by sweep j: j itself, then the earlier ones newest first, none before `first` (at the
    start of a stream a frame uses the sweeps that exist so far)."""
    return list(range(j, max(first, j - max_sweeps + 1) - 1, -1))


def schedule(n_sweeps, max_sweeps, slots):
    """The ring's order of operations for a stream of n_sweeps pushes, one frame per push:
    ("push", sweep, slot, wait_frame) - wait_frame: the last frame that read the slot's previous sweep (None: none did) -
    then ("frame", sweep, [(sweep_read, slot), ...])."""
    if slots < max_sweeps:
        raise ValueError("a ring of %d slots cannot hold the %d sweeps of a frame" % (slots, max_sweeps))
    last_reader = {}
    for j in range(n_sweeps):
        slot = j % slots
        yield ("push", j, slot, last_reader.pop(slot, None))
        reads = [(s, s % slots) for s in frame_sweeps(j, max_sweeps)]
        for _, sl in reads:
            last_reader[sl] = j
        yield ("frame", j, reads)


class SweepRing:
    """Device buffer [slots, slot_cap, raw_dim] fp32 of raw sweeps, filled on its own copy stream."""

    def __init__(self, max_sweeps, raw_dim, slot_cap, slots, device):
        import torch
        if slots < max_sweeps or slot_cap < 4 or slot_cap % 4:
            raise ValueError("need slots >= max_sweeps and slot_cap a positive multiple of 4")
        self.torch = torch
        self.max_sweeps, self.raw_dim, self.slot_cap, self.slots = int(max_sweeps), int(raw_dim), int(slot_cap), int(slots)
        self.buf = torch.zeros((slots, slot_cap, raw_dim), dtype=torch.float32, device=device)
        self._staging = [torch.empty((slot_cap, raw_dim), dtype=torch.float32).pin_memory() for _ in range(slots)]
        self.copy_stream = torch.cuda.Stream(device)
        self._pushed = [None] * slots  # event: the H2D copy into the slot is done
        self._reader = [None] * slots  # event: the last frame that read the slot is done
        self._rows = [0] * slots
        self._pose = [None] * slots
        self._time = [0.0] * slots
        self.count = 0  # sweeps pushed so far
        self.first = 0  # first sweep of the current stream

    def reset(self):
        """Start a new stream: earlier sweeps are not merged into its frames."""
        self.first = self.count

    def load(self, slot, cloud, stream):
        """Copy one raw cloud [n, raw_dim] into `slot` on `stream` (after the last frame that read the slot)."""
        torch = self.torch
        cloud = np.ascontiguousarray(cloud, np.float32)
        if cloud.ndim != 2 or cloud.shape[1] != self.raw_dim or len(cloud) > self.slot_cap:
            raise ValueError("a sweep must be [n <= %d, %d], got %s" % (self.slot_cap, self.raw_dim, cloud.shape))
        if self._pushed[slot] is not None:
            self._pushed[slot].synchronize()  # the pinned staging of this slot is free again
        n = len(cloud)
        self._staging[slot].numpy()[:n] = cloud
        with torch.cuda.stream(stream):
            if self._reader[slot] is not None:
                stream.wait_event(self._reader[slot])
            self.buf[slot, :n].copy_(self._staging[slot][:n], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(stream)
        self._pushed[slot] = ev
        self._rows[slot] = n
        return ev

    def push(self, cloud, global_from_lidar, timestamp):
        """Copy the next sweep into the ring on the copy stream; returns its index."""
        j = self.count
        slot = j % self.slots
        self.load(slot, cloud, self.copy_stream)
        self._pose[slot] = np.asarray(global_from_lidar, np.float64)
        self._time[slot] = float(timestamp)
        self.count += 1
        return j

    def describe(self, j, desc):
        """Fill desc (DESC_DTYPE [max_sweeps]) for the frame keyed by sweep j.  Returns (slots read, event of the push
        of sweep j: every earlier push is ordered before it on the copy stream)."""
        oldest = max(self.first, j - self.max_sweeps + 1)
        if not (self.first <= j < self.count and oldest >= self.count - self.slots):
            raise ValueError("sweep %d is no longer (or not yet) in the ring" % j)
        desc[:] = np.zeros(1, sm.DESC_DTYPE)
        key = j % self.slots
        read = []
        for e, s in enumerate(frame_sweeps(j, self.max_sweeps, self.first)):
            sl = s % self.slots
            if e == 0:
                sm.set_entry(desc[0], sl, self._rows[sl])
            else:
                sm.set_entry(desc[e], sl, self._rows[sl], ref_from_curr(self._pose[key], self._pose[sl]),
                             self._time[key] - self._time[sl])
            read.append(sl)
        return read, self._pushed[key]

    def mark_read(self, slots, event):
        """`event` completes after the frame that read `slots` (a later record of the same event is also fine)."""
        for sl in slots:
            self._reader[sl] = event
