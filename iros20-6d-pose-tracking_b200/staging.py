"""Decoding ahead of the device through one ring of pinned staging sets.

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
