"""Decoding ahead of the device through one ring of pinned staging sets, and (VideoSink) writing device frames to video files
behind it through another.

A StagingRing holds `depth` sets of pinned host tensors and one set of device tensors with the same names.  Its uploads()
runs the caller's decode jobs in a thread pool, each item's jobs writing into one host set, and copies every item into the
device set in order, on the current stream, while up to `depth` items decode ahead of the one being consumed.  The device
set keeps its addresses for the ring's lifetime, so steps keyed by their device pointers (tracking, validation) replay their
CUDA graphs.

The one rule every caller relies on lives here: a host set is handed to a decode job only after the last asynchronous copy
out of it has completed.  Rewriting it earlier would not fail; the device would read an item that is half old and half new.
"""
from collections import deque
from concurrent.futures import ThreadPoolExecutor

import torch


class StagingRing:
    def __init__(self, spec, depth, device):
        """spec: {name: (shape, dtype)} of one set.  depth: the number of pinned host sets, at least 1."""
        self.host = [{k: torch.empty(shape, dtype=dt, pin_memory=True) for k, (shape, dt) in spec.items()} for _ in range(depth)]
        self.dev = {k: torch.empty(shape, dtype=dt, device=device) for k, (shape, dt) in spec.items()}
        self.device = torch.device(device)
        self._uploaded = [torch.cuda.Event() for _ in range(depth)]      # recorded after the last upload from each host set

    def uploads(self, items, workers, rows=None):
        """Yields, for each item in order, the return values of its jobs, once its upload into `dev` is queued on the current
        stream.  An item is a list of jobs (fn, *args); each runs as fn(host set, *args) on one of `workers` threads.  rows[k]
        (rows None: every row) is how many leading rows item k uploads.  A job's exception is raised when its item is reached.
        The pool is shut down, its running jobs finished and its queued ones cancelled, when the iteration ends, raises or is
        closed."""
        depth = len(self.host)
        pool = ThreadPoolExecutor(max_workers=workers)
        pending = deque()
        submitted = 0
        try:
            for k in range(len(items)):
                while submitted < min(k + depth, len(items)):                # item j decodes into host set j % depth
                    h = self.host[submitted % depth]
                    self._uploaded[submitted % depth].synchronize()           # the set's last upload has left it
                    pending.append([pool.submit(fn, h, *args) for fn, *args in items[submitted]])
                    submitted += 1
                values = [f.result() for f in pending.popleft()]
                n = None if rows is None else rows[k]
                stream = torch.cuda.current_stream(self.device)
                for name, d in self.dev.items():
                    d[:n].copy_(self.host[k % depth][name][:n], non_blocking=True)
                self._uploaded[k % depth].record(stream)
                yield values
        finally:
            pool.shutdown(wait=True, cancel_futures=True)


class VideoSink:
    """The other direction: device frames downloaded through `depth` pinned host sets and written to mp4 files by one writer
    thread.  put() queues a non-blocking device-to-host copy of one item on the current stream, records an event after it, and
    hands the host set to the writer, which waits on that event and appends frame j of the item to video paths[j]
    (cv2.VideoWriter, mp4v at `fps`), in the order put() was called.  A host set is rewritten only after the writer has written
    its frames, so the stream never waits on the writer; put() waits when all `depth` sets are still being written.  A writer
    exception is raised by the next put() or by close().  close() (also on an exception) writes what was queued and releases
    every file, so each one is complete when it returns."""

    def __init__(self, shape, depth, device, fps=30):
        """shape: (most frames per item, H, W, 3) uint8 BGR frames."""
        self.host = [torch.empty(shape, dtype=torch.uint8, pin_memory=True) for _ in range(depth)]
        self.device = torch.device(device)
        self.fps = fps
        self._copied = [torch.cuda.Event() for _ in range(depth)]
        self._written = [None] * depth                                  # the writer's future for each host set
        self._writers = {}                                              # path -> open cv2.VideoWriter
        self._pool = ThreadPoolExecutor(max_workers=1)
        self._next = 0

    def put(self, frames, paths, last=False):
        """frames: uint8 CUDA (k, H, W, 3); frame j is the next frame of video paths[j].  last: those videos end with it and are
        released once it is written."""
        for f in self._written:                                         # a failed write surfaces at the next frame
            if f is not None and f.done():
                f.result()
        slot = self._next % len(self.host)
        if self._written[slot] is not None:
            self._written[slot].result()                                # the set's frames are written
        k = int(frames.shape[0])
        self.host[slot][:k].copy_(frames, non_blocking=True)
        self._copied[slot].record(torch.cuda.current_stream(self.device))
        self._written[slot] = self._pool.submit(self._write, slot, list(paths), last)
        self._next += 1

    def _write(self, slot, paths, last):
        import cv2
        self._copied[slot].synchronize()
        for j, path in enumerate(paths):
            w = self._writers.get(path)
            if w is None:
                h, wd = self.host[slot].shape[1:3]
                w = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*'mp4v'), self.fps, (int(wd), int(h)))
                if not w.isOpened():
                    raise OSError('cannot open a video writer for %s' % path)
                self._writers[path] = w
            w.write(self.host[slot][j].numpy())
        if last:
            for path in paths:
                self._writers.pop(path).release()

    def close(self):
        try:
            for f in self._written:
                if f is not None:
                    f.result()
        finally:
            self._pool.shutdown(wait=True, cancel_futures=True)
            for w in self._writers.values():
                w.release()
            self._writers.clear()
